/* tests/oracle_proje/kge_oracle_proje.c — TEST INFRASTRUCTURE: scalar C restatement of ProjE_pointwise
 * (pykg2vec/models/projection.py:128-257) in the canonical arithmetic of pykg2vec_b200/csrc/kge_proje.cuh: the
 * trunk, the per-entry logit / loss terms / g of the training step, and its gradients.  The CUDA path must agree
 * with it bit for bit on x, the logits and g.  A second path evaluates the same step in double (libm tanh / exp
 * / log) as the tolerance reference of the loss and the gradients.  Built with gcc -O2 -ffp-contract=off
 * -fno-fast-math -mfma (fmaf() is explicit, nothing else is contracted) by tests/proje_util.py.  Nothing in
 * pykg2vec_b200/ can reach it. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* kge_proje_t of include/kge_b200.h */
typedef struct kge_proje {
  int32_t hidden_size;
  int64_t num_ent, num_rel;
  const float* ent; const float* rel;
  const float* bc1; const float* De1; const float* Dr1;
  const float* bc2; const float* De2; const float* Dr2;
} kge_proje_t;

/* canonical exp / sigmoid / tanh / log: the Cephes forms of oracle/kge_oracle.c */
static float c_expf(float x) {
  x = fminf(fmaxf(x, -87.0f), 87.0f);
  const float k = rintf(x * 1.44269504088896341f);
  float r = fmaf(-k, 0.693359375f, x);
  r = fmaf(-k, -2.12194440e-4f, r);
  float p = fmaf(r, 1.9875691500e-4f, 1.3981999507e-3f);
  p = fmaf(p, r, 8.3334519073e-3f);
  p = fmaf(p, r, 4.1665795894e-2f);
  p = fmaf(p, r, 1.6666665459e-1f);
  p = fmaf(p, r, 5.0000001201e-1f);
  const float y = fmaf(p, r * r, r) + 1.0f;
  union { uint32_t u; float f; } two_k;
  two_k.u = (uint32_t)((int)k + 127) << 23;
  return y * two_k.f;
}
static float c_sigmoidf(float x) { return 1.0f / (1.0f + c_expf(-x)); }
static float c_tanhf(float x) {
  const float ax = fabsf(x);
  if (ax < 0.625f) {
    const float z = x * x;
    float p = fmaf(-5.70498872745e-3f, z, 2.06390887954e-2f);
    p = fmaf(p, z, -5.37397155531e-2f);
    p = fmaf(p, z, 1.33314422036e-1f);
    p = fmaf(p, z, -3.33332819422e-1f);
    return fmaf(p * z, x, x);
  }
  const float e = c_expf(2.0f * ax);
  const float t = 1.0f - 2.0f * (1.0f / (e + 1.0f));
  return x < 0.0f ? -t : t;
}
static float c_logf(float x) {
  if (!(x > 0.0f)) return x == 0.0f ? -INFINITY : NAN;
  if (isinf(x)) return x;
  int e = 0;
  if (x < 1.17549435e-38f) { x = x * 8388608.0f; e = -23; }
  union { float f; uint32_t u; } v; v.f = x;
  e += (int)((v.u >> 23) & 0xff) - 126;
  v.u = (v.u & 0x007fffffu) | 0x3f000000u;
  float m = v.f;
  if (m < 0.707106781186547524f) { e -= 1; m = (m + m) - 1.0f; } else { m = m - 1.0f; }
  const float z = m * m;
  float y = fmaf(7.0376836292e-2f, m, -1.1514610310e-1f);
  y = fmaf(y, m, 1.1676998740e-1f);
  y = fmaf(y, m, -1.2420140846e-1f);
  y = fmaf(y, m, 1.4249322787e-1f);
  y = fmaf(y, m, -1.6668057665e-1f);
  y = fmaf(y, m, 2.0000714765e-1f);
  y = fmaf(y, m, -2.4999993993e-1f);
  y = fmaf(y, m, 3.3333331174e-1f);
  y = (y * m) * z;
  const float fe = (float)e;
  y = fmaf(-2.12194440e-4f, fe, y);
  y = fmaf(-0.5f, z, y);
  float r = m + y;
  r = fmaf(0.693359375f, fe, r);
  return r;
}

static void dir_tables(const kge_proje_t* p, int d, const float** De, const float** Dr, const float** bc) {
  *De = d ? p->De2 : p->De1; *Dr = d ? p->Dr2 : p->Dr1; *bc = d ? p->bc2 : p->bc1;
}

/* x[q, j] = tanh(fadd(fadd(fmul(e, De), fmul(r, Dr)), bc)) [* noise[q, j]]; direction 0 = f1, 1 = f2 */
int kgeo_proje_trunk(const kge_proje_t* p, int dir, const int64_t* e, const int64_t* r, int64_t Q,
                     const float* noise, float* x) {
  const int k = p->hidden_size;
  const float *De, *Dr, *bc;
  dir_tables(p, dir, &De, &Dr, &bc);
  for (int64_t q = 0; q < Q; ++q)
    for (int j = 0; j < k; ++j) {
      const float ev = p->ent[e[q] * k + j], rv = p->rel[r[q] * k + j];
      float v = c_tanhf((ev * De[j] + rv * Dr[j]) + bc[j]);
      if (noise) v = v * noise[q * k + j];
      x[q * k + j] = v;
    }
  return 0;
}

/* The training step of kge_proje_train_step over both directions (labels[d] NULL: skipped).
 * fp64 = 0: the canonical fp32 arithmetic per entry; d loss / d x and the gradients are fp32 sums in ascending
 *           entity order, the loss a double sum of the fp32 terms.  logit_out / g_out ([2][B][N], may be NULL)
 *           receive the logit and g of every labelled entry (others untouched).
 * fp64 = 1: the same formulas in double with libm tanh / exp / log (clamps and their zero-gradient branches
 *           included); the gradients are accumulated in double and added to grads[] once, rounded to fp32.
 * grads[8] (parameter_list order: ent, rel, bc1, De1, Dr1, bc2, De2, Dr2; each may be NULL) are accumulated. */
int kgeo_proje_step(const kge_proje_t* p, const int64_t* ids0, const int64_t* ids1, const int64_t* r, int64_t B,
                    const float* lab0, const float* lab1, const float* noise0, const float* noise1, int fp64,
                    float* logit_out, float* g_out, float* const* grads, double* loss_out) {
  const int k = p->hidden_size;
  const int64_t N = p->num_ent, R = p->num_rel;
  const int64_t sizes[8] = {N * k, R * k, k, k, k, k, k, k};
  double* acc[8];
  for (int i = 0; i < 8; ++i) acc[i] = fp64 ? (double*)calloc((size_t)sizes[i], sizeof(double)) : NULL;
  double* tx = (double*)malloc(sizeof(double) * (size_t)k);
  double* xx = (double*)malloc(sizeof(double) * (size_t)k);
  double* gxd = (double*)malloc(sizeof(double) * (size_t)k);
  float* tf = (float*)malloc(sizeof(float) * (size_t)k);
  float* xf = (float*)malloc(sizeof(float) * (size_t)k);
  float* gxf = (float*)malloc(sizeof(float) * (size_t)k);
  double loss = 0.0;
  for (int d = 0; d < 2; ++d) {
    const float* lab = d ? lab1 : lab0;
    const int64_t* ids = d ? ids1 : ids0;
    const float* noise = d ? noise1 : noise0;
    if (!lab) continue;
    const float *De, *Dr, *bc;
    dir_tables(p, d, &De, &Dr, &bc);
    const int gi_bc = d ? 5 : 2, gi_De = d ? 6 : 3, gi_Dr = d ? 7 : 4;
    for (int64_t b = 0; b < B; ++b) {
      const float* er = p->ent + ids[b] * k;
      const float* rr = p->rel + r[b] * k;
      const float* nz = noise ? noise + b * k : NULL;
      for (int j = 0; j < k; ++j) {
        if (fp64) {
          tx[j] = tanh((double)er[j] * De[j] + (double)rr[j] * Dr[j] + bc[j]);
          xx[j] = nz ? tx[j] * nz[j] : tx[j];
          gxd[j] = 0.0;
        } else {
          tf[j] = c_tanhf((er[j] * De[j] + rr[j] * Dr[j]) + bc[j]);
          xf[j] = nz ? tf[j] * nz[j] : tf[j];
          gxf[j] = 0.0f;
        }
      }
      for (int64_t n = 0; n < N; ++n) {
        const float y = lab[b * N + n];
        if (y == 0.0f) continue;
        const float* en = p->ent + n * k;
        const float wl = y > 0.0f ? y : 0.0f, wr = -y > 0.0f ? -y : 0.0f;
        if (fp64) {
          double z = 0.0;
          for (int j = 0; j < k; ++j) z += xx[j] * en[j];
          const double s = 1.0 / (1.0 + exp(-z)), o = 1.0 - s;
          const double c1 = fmin(fmax(s, 1e-10), 1.0), c2 = fmin(fmax(o, 1e-10), 1.0);
          loss -= log(c1) * wl + log(c2) * wr;
          const double ds = ((s >= 1e-10 && s <= 1.0) ? -wl / c1 : 0.0) + ((o >= 1e-10 && o <= 1.0) ? wr / c2 : 0.0);
          const double g = ds * o * s;
          for (int j = 0; j < k; ++j) {
            gxd[j] += g * en[j];
            acc[0][n * k + j] += g * xx[j];
          }
        } else {
          float z = 0.0f;
          for (int j = 0; j < k; ++j) z = fmaf(xf[j], en[j], z);
          const float s = c_sigmoidf(z), o = 1.0f - s;
          const float c1 = fminf(fmaxf(s, 1e-10f), 1.0f), c2 = fminf(fmaxf(o, 1e-10f), 1.0f);
          loss -= (double)(c_logf(c1) * wl + c_logf(c2) * wr);
          const float gl = (s >= 1e-10f && s <= 1.0f) ? -wl / c1 : 0.0f;
          const float gr = (o >= 1e-10f && o <= 1.0f) ? wr / c2 : 0.0f;
          const float g = ((gl + gr) * o) * s;
          if (logit_out) logit_out[(d * B + b) * N + n] = z;
          if (g_out) g_out[(d * B + b) * N + n] = g;
          if (g == 0.0f) continue;
          for (int j = 0; j < k; ++j) {
            gxf[j] = fmaf(g, en[j], gxf[j]);
            if (grads[0]) grads[0][n * k + j] += g * xf[j];
          }
        }
      }
      for (int j = 0; j < k; ++j) {
        if (fp64) {
          const double gp = (nz ? gxd[j] * nz[j] : gxd[j]) * (1.0 - tx[j] * tx[j]);
          acc[0][ids[b] * k + j] += gp * De[j];
          acc[1][r[b] * k + j] += gp * Dr[j];
          acc[gi_De][j] += gp * er[j];
          acc[gi_Dr][j] += gp * rr[j];
          acc[gi_bc][j] += gp;
        } else {
          const float gp = (nz ? gxf[j] * nz[j] : gxf[j]) * (1.0f - tf[j] * tf[j]);
          if (grads[0]) grads[0][ids[b] * k + j] += gp * De[j];
          if (grads[1]) grads[1][r[b] * k + j] += gp * Dr[j];
          if (grads[gi_De]) grads[gi_De][j] += gp * er[j];
          if (grads[gi_Dr]) grads[gi_Dr][j] += gp * rr[j];
          if (grads[gi_bc]) grads[gi_bc][j] += gp;
        }
      }
    }
  }
  for (int i = 0; i < 8; ++i) {
    if (acc[i] && grads[i])
      for (int64_t m = 0; m < sizes[i]; ++m) grads[i][m] += (float)acc[i][m];
    free(acc[i]);
  }
  free(tx); free(xx); free(gxd); free(tf); free(xf); free(gxf);
  *loss_out = loss;
  return 0;
}

/* get_reg (projection.py:189-192): lmbda * sum |w| over n floats, in double; grad (may be NULL) += lmbda sign(w)
 * in fp32 (sign(0) = 0) */
double kgeo_reg_l1(const float* w, int64_t n, float lmbda, float* grad) {
  double s = 0.0;
  for (int64_t i = 0; i < n; ++i) {
    s += fabs((double)w[i]);
    if (grad) grad[i] += w[i] > 0.0f ? lmbda : (w[i] < 0.0f ? -lmbda : 0.0f);
  }
  return s * (double)lmbda;
}
