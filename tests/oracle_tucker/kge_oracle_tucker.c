/* tests/oracle_tucker/kge_oracle_tucker.c — TEST ORACLE: a scalar restatement of TuckER's trunk
 * (pykg2vec/models/projection.py:310-336) in the canonical arithmetic of DESIGN.md §3 (TuckER), against which the
 * kernels of pykg2vec_b200/csrc/kge_tucker.cuh are compared: the forward bit for bit, the backward (computed here
 * in double from the fp32 forward values) within rounding.  Build: gcc -O2 -ffp-contract=off -mfma (fmaf explicit).
 *
 *   cores    M[u][c] = one fmaf chain over k = 0 .. d2-1 from 0 of rel[ids[u]][k] * W[k][c]
 *   sumsq    RSUM: 8 partials, element j -> partial (j >> 2) & 7 in increasing j by fmaf, then
 *            ((p0+p4) + (p2+p6)) + ((p1+p5) + (p3+p7))   (the xor butterfly 4, 2, 1 seen from lane 0)
 *   ehat[i]  = (ent[e][i] / max(sqrtf(sumsq), 1e-12)) * noise0[i]
 *   xpre[j]  = one fmaf chain over i = 0 .. d1-1 from 0 of ehat[i] * (m1[i][j] * M[i][j]); no mask: ehat[i] * M[i][j]
 *   x[j]     = (xpre[j] / max(sqrtf(sumsq(xpre)), 1e-12)) * noise2[j]
 *   m1       explicit: noise1.  counter: word 0 of Philox-4x32-10, key (seed lo, seed hi), counter
 *            (lo, hi of offset + (q*d1 + i)*d1 + j, 0x7475636b, 0); kept iff >= ceil(p 2^32) (clamped to 2^32 - 1),
 *            kept value 1 / (float)(1 - p); p >= 1 drops everything. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>

typedef struct {
  int32_t d1, d2;
  int64_t num_ent, num_rel;
  const float* ent; const float* rel; const float* W;
} kge_tucker_t;

static uint32_t philox(uint64_t seed, uint64_t ctr) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = 0x7475636bu, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    c1 = (uint32_t)p1; c3 = (uint32_t)p0; c0 = n0; c2 = n2;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

static void mask_params(float p, uint32_t* thresh, float* scale) {
  if (p >= 1.0f) { *thresh = 0xffffffffu; *scale = 0.f; return; }
  if (p == 0.f) { *thresh = 0u; *scale = 1.0f; return; }
  const double t = ceil((double)p * 4294967296.0);
  *thresh = t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
  *scale = 1.0f / (float)(1.0 - (double)p);
}

/* mode 0 none, 1 explicit, 2 counter */
typedef struct { int mode; const float* noise1; uint64_t seed, offset; uint32_t thresh; float scale; } mask_t;

static float mask_at(const mask_t* m, int64_t idx) {
  if (m->mode == 1) return m->noise1[idx];
  return philox(m->seed, m->offset + (uint64_t)idx) >= m->thresh ? m->scale : 0.f;
}

static mask_t make_mask(int mode, const float* noise1, uint64_t seed, uint64_t offset, float p) {
  mask_t m = {mode, noise1, seed, offset, 0u, 1.0f};
  if (mode == 2) {
    if (p == 0.f) m.mode = 0;
    mask_params(p, &m.thresh, &m.scale);
  }
  return m;
}

static float rsum(const float* a, const float* b, int n) {
  float p[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int j = 0; j < n; ++j) p[(j >> 2) & 7] = fmaf(a[j], b[j], p[(j >> 2) & 7]);
  return ((p[0] + p[4]) + (p[2] + p[6])) + ((p[1] + p[5]) + (p[3] + p[7]));
}

int kgeo_tucker_mask1(uint64_t seed, uint64_t offset, float p, int64_t n, float* out) {
  mask_t m = {2, 0, seed, offset, 0u, 1.0f};
  mask_params(p, &m.thresh, &m.scale);
  for (int64_t i = 0; i < n; ++i) out[i] = mask_at(&m, i);
  return 0;
}

int kgeo_tucker_cores(const kge_tucker_t* p, const int64_t* ids, int64_t U, float* M) {
  const int64_t dd = (int64_t)p->d1 * p->d1;
  for (int64_t u = 0; u < U; ++u)
    for (int64_t c = 0; c < dd; ++c) {
      float acc = 0.f;
      for (int k = 0; k < p->d2; ++k) acc = fmaf(p->rel[ids[u] * p->d2 + k], p->W[k * dd + c], acc);
      M[u * dd + c] = acc;
    }
  return 0;
}

int kgeo_tucker_trunk_fwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                          const float* noise0, int mode, const float* noise1, uint64_t seed, uint64_t offset,
                          float pdrop, const float* noise2, float* x, float* xpre, float* nrm) {
  const int d1 = p->d1;
  const int64_t dd = (int64_t)d1 * d1;
  const mask_t m = make_mask(mode, noise1, seed, offset, pdrop);
  float* eh = (float*)malloc(sizeof(float) * 2 * d1);
  float* xp = eh + d1;
  for (int64_t q = 0; q < Q; ++q) {
    const float* er = p->ent + e[q] * d1;
    const float den = fmaxf(sqrtf(rsum(er, er, d1)), 1e-12f);
    for (int i = 0; i < d1; ++i) {
      eh[i] = er[i] / den;
      if (noise0) eh[i] = eh[i] * noise0[q * d1 + i];
    }
    const float* Mq = M + slot[q] * dd;
    for (int j = 0; j < d1; ++j) {
      float acc = 0.f;
      for (int i = 0; i < d1; ++i) {
        const int64_t o = (int64_t)i * d1 + j;
        acc = m.mode ? fmaf(eh[i], mask_at(&m, q * dd + o) * Mq[o], acc) : fmaf(eh[i], Mq[o], acc);
      }
      xp[j] = acc;
    }
    const float n2 = sqrtf(rsum(xp, xp, d1));
    for (int j = 0; j < d1; ++j) {
      float v = xp[j] / fmaxf(n2, 1e-12f);
      if (noise2) v = v * noise2[q * d1 + j];
      x[q * d1 + j] = v;
      if (xpre) xpre[q * d1 + j] = xp[j];
    }
    if (nrm) nrm[q] = n2;
  }
  free(eh);
  return 0;
}

/* y = v / max(n, eps), n = ||v||: dv = (dy - yhat (dy . yhat)) / n while n > eps, else dy / eps */
static void norm_bwd(const double* dy, const double* yhat, double n, int d, double* dv) {
  double dot = 0.0;
  for (int j = 0; j < d; ++j) dot += dy[j] * yhat[j];
  for (int j = 0; j < d; ++j) dv[j] = n > 1e-12 ? (dy[j] - yhat[j] * dot) / n : dy[j] / 1e-12;
}

/* backward of the trunk in double from the fp32 parameters: gent [N, d1] and dM [U, d1*d1] (double, accumulated;
 * each may be NULL) */
int kgeo_tucker_trunk_bwd(const kge_tucker_t* p, const float* M, const int64_t* e, const int64_t* slot, int64_t Q,
                          const float* noise0, int mode, const float* noise1, uint64_t seed, uint64_t offset,
                          float pdrop, const float* noise2, const float* gx, double* gent, double* dM) {
  const int d1 = p->d1;
  const int64_t dd = (int64_t)d1 * d1;
  const mask_t m = make_mask(mode, noise1, seed, offset, pdrop);
  double* buf = (double*)malloc(sizeof(double) * 7 * d1);
  double *en = buf, *eh = buf + d1, *xp = buf + 2 * d1, *xh = buf + 3 * d1, *g = buf + 4 * d1, *de = buf + 5 * d1,
         *t = buf + 6 * d1;
  for (int64_t q = 0; q < Q; ++q) {
    const float* er = p->ent + e[q] * d1;
    double n1 = 0.0, n2 = 0.0;
    for (int i = 0; i < d1; ++i) n1 += (double)er[i] * er[i];
    n1 = sqrt(n1);
    for (int i = 0; i < d1; ++i) {
      en[i] = er[i] / fmax(n1, 1e-12);
      eh[i] = noise0 ? en[i] * noise0[q * d1 + i] : en[i];
    }
    const float* Mq = M + slot[q] * dd;
    for (int j = 0; j < d1; ++j) {
      double acc = 0.0;
      for (int i = 0; i < d1; ++i) {
        const int64_t o = (int64_t)i * d1 + j;
        acc += eh[i] * (m.mode ? (double)mask_at(&m, q * dd + o) : 1.0) * Mq[o];
      }
      xp[j] = acc;
      n2 += acc * acc;
    }
    n2 = sqrt(n2);
    for (int j = 0; j < d1; ++j) {
      xh[j] = xp[j] / fmax(n2, 1e-12);
      t[j] = noise2 ? (double)gx[q * d1 + j] * noise2[q * d1 + j] : (double)gx[q * d1 + j];
    }
    norm_bwd(t, xh, n2, d1, g);
    for (int i = 0; i < d1; ++i) {
      double acc = 0.0;
      for (int j = 0; j < d1; ++j) {
        const int64_t o = (int64_t)i * d1 + j;
        const double mv = m.mode ? (double)mask_at(&m, q * dd + o) : 1.0;
        acc += mv * Mq[o] * g[j];
        if (dM) dM[slot[q] * dd + o] += eh[i] * mv * g[j];
      }
      de[i] = noise0 ? acc * noise0[q * d1 + i] : acc;
    }
    if (gent) {
      norm_bwd(de, en, n1, d1, t);
      for (int i = 0; i < d1; ++i) gent[e[q] * d1 + i] += t[i];
    }
  }
  free(buf);
  return 0;
}

/* gW[k][c] += sum_u rel[ids[u]][k] dM[u][c];  grel[ids[u]][k] += sum_c dM[u][c] W[k][c]   (double, accumulated) */
int kgeo_tucker_cores_bwd(const kge_tucker_t* p, const int64_t* ids, int64_t U, const double* dM, double* grel,
                          double* gW) {
  const int64_t dd = (int64_t)p->d1 * p->d1;
  for (int64_t u = 0; u < U; ++u)
    for (int k = 0; k < p->d2; ++k) {
      const double rv = p->rel[ids[u] * p->d2 + k];
      double acc = 0.0;
      for (int64_t c = 0; c < dd; ++c) {
        if (gW) gW[k * dd + c] += rv * dM[u * dd + c];
        acc += dM[u * dd + c] * p->W[k * dd + c];
      }
      if (grel) grel[ids[u] * p->d2 + k] += acc;
    }
  return 0;
}
