/* tests/oracle_interacte_train/kge_oracle_interacte_train.c — TEST INFRASTRUCTURE: CPU oracle of InteractE's
 * training-mode trunk (pykg2vec_b200/csrc/kge_interacte_train.cuh, pykg2vec/models/projection.py:425-442 with
 * self.training == True).
 *
 * kgeo_interacte_train_fwd restates the kernels' canonical arithmetic in scalar C with explicit fmaf and no contraction
 * (-ffp-contract=off): bn0's per-query partials as one CTA sum per image in pixel order (256 per-thread chains, xor
 * butterfly inside each warp, warp sums in ascending order), bn1's as warp sums per channel (32 lane chains, butterfly),
 * the partials combined in ascending query order, the circular conv as ks*ks sequential fmaf from 0 (row u, then column
 * v), the Linear layer's 512-feature slices added in order, bn2's two passes.  x and the running statistics must equal
 * the kernels' bit for bit.  Queries are independent within a phase, so the OpenMP loops do not change a bit.
 *
 * kgeo_interacte_train_bwd64 is the same trunk in double, forward and backward (the analytic BatchNorm, circular conv,
 * Linear and permutation backward): the yardstick of the kernels' backward. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/kge_b200.h"

#define NT 256 /* CONVE_TR_THREADS */

static float butterfly32(float* a) {
  for (int off = 16; off; off >>= 1) {
    float b[32];
    for (int l = 0; l < 32; ++l) b[l] = a[l] + a[l ^ off];
    memcpy(a, b, sizeof b);
  }
  return a[0];
}

static float cta_combine(float* t) {
  float s = butterfly32(t);
  for (int k = 1; k < NT / 32; ++k) s = s + butterfly32(t + 32 * k);
  return s;
}

static float cta_sum(const float* v, int n) {
  float t[NT];
  for (int i = 0; i < NT; ++i) t[i] = 0.0f;
  for (int i = 0; i < n; ++i) t[i % NT] = t[i % NT] + v[i];
  return cta_combine(t);
}

static float cta_m2(const float* v, int n, float m) {
  float t[NT];
  for (int i = 0; i < NT; ++i) t[i] = 0.0f;
  for (int i = 0; i < n; ++i) { const float d = v[i] - m; t[i % NT] = fmaf(d, d, t[i % NT]); }
  return cta_combine(t);
}

static void warp_stats(const float* v, int n, float* s_out, float* m2_out) {
  float a[32];
  for (int l = 0; l < 32; ++l) a[l] = 0.0f;
  for (int p = 0; p < n; ++p) a[p % 32] = a[p % 32] + v[p];
  const float s = butterfly32(a);
  const float m = s / (float)n;
  for (int l = 0; l < 32; ++l) a[l] = 0.0f;
  for (int p = 0; p < n; ++p) { const float d = v[p] - m; a[p % 32] = fmaf(d, d, a[p % 32]); }
  *s_out = s;
  *m2_out = butterfly32(a);
}

static void bn_stats(const float* part, int64_t Q, int64_t B, int C, int c, float nq, float eps, float mom, float* st,
                     float* rmean, float* rvar) {
  const int64_t G = Q / B;
  const float n = (float)B * nq;
  for (int64_t g = 0; g < G; ++g) {
    const float* pp = part + (g * B * C + c) * 2;
    float S = 0.0f;
    for (int64_t i = 0; i < B; ++i) S = S + pp[i * C * 2];
    const float mean = S / n;
    float M2 = 0.0f;
    for (int64_t i = 0; i < B; ++i) {
      const float d = pp[i * C * 2] / nq - mean;
      M2 = M2 + fmaf(nq * d, d, pp[i * C * 2 + 1]);
    }
    const float var = M2 / n;
    st[(g * C + c) * 2] = mean;
    st[(g * C + c) * 2 + 1] = 1.0f / sqrtf(var + eps);
    if (rmean) {
      rmean[c] = fmaf(mom, mean, (1.0f - mom) * rmean[c]);
      rvar[c] = fmaf(mom, (var * n) / (n - 1.0f), (1.0f - mom) * rvar[c]);
    }
  }
}

static float bn_apply(float v, float mean, float invstd, float w, float b) { return fmaf((v - mean) * invstd, w, b); }

static int wrap(int i, int n) { return i < 0 ? i + n : (i >= n ? i - n : i); }

int kgeo_interacte_train_fwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                             const float* n0, const float* n1, const float* n2, float* x) {
  const int P = p->feature_permutation, F = p->num_filters, ks = p->kernel_size, pad = ks / 2;
  const int H = 2 * p->reshape_width, W = p->reshape_height, HW = H * W, k = HW / 2, C1 = P * F;
  const int64_t Fw = (int64_t)C1 * HW, G = Q / B;
  float* img = (float*)malloc(sizeof(float) * (size_t)(Q * P * HW));
  float* z1 = (float*)malloc(sizeof(float) * (size_t)(Q * Fw));
  float* hp = (float*)malloc(sizeof(float) * (size_t)(Q * k));
  float* part0 = (float*)malloc(sizeof(float) * (size_t)(Q * P * 2));
  float* part1 = (float*)malloc(sizeof(float) * (size_t)(Q * C1 * 2));
  float* st0 = (float*)malloc(sizeof(float) * (size_t)(G * P * 2));
  float* st1 = (float*)malloc(sizeof(float) * (size_t)(G * C1 * 2));
  for (int64_t q = 0; q < Q; ++q)
    for (int pp = 0; pp < P; ++pp) {
      float* im = img + (q * P + pp) * HW;
      for (int i = 0; i < HW; ++i) {
        const int64_t c = p->perm[(int64_t)pp * HW + i];
        im[i] = c < k ? p->ent[e[q] * k + c] : p->rel[r[q] * k + (c - k)];
      }
      const float s = cta_sum(im, HW);
      part0[(q * P + pp) * 2] = s;
      part0[(q * P + pp) * 2 + 1] = cta_m2(im, HW, s / (float)HW);
    }
  for (int c = 0; c < P; ++c)
    bn_stats(part0, Q, B, P, c, (float)HW, p->bn0_eps, p->bn0_momentum, st0, p->bn0_mean, p->bn0_var);
#pragma omp parallel for schedule(static)
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    float* v = (float*)malloc(sizeof(float) * (size_t)(P * HW));
    for (int pp = 0; pp < P; ++pp)
      for (int i = 0; i < HW; ++i) {
        const int64_t at = (q * P + pp) * HW + i;
        const float y = bn_apply(img[at], st0[(g * P + pp) * 2], st0[(g * P + pp) * 2 + 1], p->bn0_weight[pp],
                                 p->bn0_bias[pp]);
        v[pp * HW + i] = n0 ? y * n0[at] : y;
      }
    float* zq = z1 + q * Fw;
    for (int pp = 0; pp < P; ++pp)
      for (int f = 0; f < F; ++f)
        for (int i = 0; i < H; ++i)
          for (int j = 0; j < W; ++j) {
            float acc = 0.0f;
            for (int u = 0; u < ks; ++u)
              for (int vv = 0; vv < ks; ++vv)
                acc = fmaf(p->conv_filt[((int64_t)f * ks + u) * ks + vv],
                           v[pp * HW + wrap(i + u - pad, H) * W + wrap(j + vv - pad, W)], acc);
            zq[(int64_t)(pp * F + f) * HW + i * W + j] = acc;
          }
    for (int c = 0; c < C1; ++c)
      warp_stats(zq + (int64_t)c * HW, HW, &part1[(q * C1 + c) * 2], &part1[(q * C1 + c) * 2 + 1]);
    free(v);
  }
  for (int c = 0; c < C1; ++c)
    bn_stats(part1, Q, B, C1, c, (float)HW, p->bn1_eps, p->bn1_momentum, st1, p->bn1_mean, p->bn1_var);
#pragma omp parallel for schedule(static)
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    float* feat = (float*)malloc(sizeof(float) * (size_t)Fw);
    for (int64_t o = 0; o < Fw; ++o) {
      const int c = (int)(o / HW);
      float y = bn_apply(z1[q * Fw + o], st1[(g * C1 + c) * 2], st1[(g * C1 + c) * 2 + 1], p->bn1_weight[c],
                         p->bn1_bias[c]);
      y = fmaxf(y, 0.0f);
      feat[o] = n1 ? y * n1[q * C1 + c] : y;
    }
    for (int n = 0; n < k; ++n) {   /* Linear: per-slice fmaf chains, slice sums added in order */
      const float* fw = p->fc_weight + (int64_t)n * Fw;
      float total = 0.0f;
      for (int64_t f0 = 0; f0 < Fw; f0 += 512) {
        const int64_t f1 = f0 + 512 < Fw ? f0 + 512 : Fw;
        float acc = 0.0f;
        for (int64_t f = f0; f < f1; ++f) acc = fmaf(feat[f], fw[f], acc);
        total = (f0 == 0) ? acc : total + acc;
      }
      total = total + p->fc_bias[n];
      hp[q * k + n] = n2 ? total * n2[q * k + n] : total;
    }
    free(feat);
  }
  for (int j = 0; j < k; ++j) {   /* bn2: two passes per feature over each group's rows */
    const float nB = (float)B, wj = p->bn2_weight[j], bj = p->bn2_bias[j];
    for (int64_t g = 0; g < G; ++g) {
      float S = 0.0f;
      for (int64_t i = g * B; i < (g + 1) * B; ++i) S = S + hp[i * k + j];
      const float mean = S / nB;
      float M2 = 0.0f;
      for (int64_t i = g * B; i < (g + 1) * B; ++i) { const float d = hp[i * k + j] - mean; M2 = fmaf(d, d, M2); }
      const float var = M2 / nB, invstd = 1.0f / sqrtf(var + p->bn2_eps);
      if (p->bn2_mean) {
        p->bn2_mean[j] = fmaf(p->bn2_momentum, mean, (1.0f - p->bn2_momentum) * p->bn2_mean[j]);
        p->bn2_var[j] = fmaf(p->bn2_momentum, (var * nB) / (nB - 1.0f), (1.0f - p->bn2_momentum) * p->bn2_var[j]);
      }
      for (int64_t i = g * B; i < (g + 1) * B; ++i) x[i * k + j] = fmaxf(bn_apply(hp[i * k + j], mean, invstd, wj, bj), 0.0f);
    }
  }
  free(img); free(z1); free(hp); free(part0); free(part1); free(st0); free(st1);
  return 0;
}

/* ---- fp64 forward + backward ------------------------------------------------------------------------------------ */

/* grads: 11 buffers in kge_interacte_train_bwd order (ent, rel, bn0.w, bn0.b, conv_filt, bn1.w, bn1.b, fc.w, fc.b,
 * bn2.w, bn2.b), ACCUMULATED; gx [Q, k]; x64 (may be NULL) receives the fp64 forward's x */
int kgeo_interacte_train_bwd64(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q,
                               int64_t B, const float* n0, const float* n1, const float* n2, const double* gx,
                               double* const* grads, double* x64) {
  const int P = p->feature_permutation, F = p->num_filters, ks = p->kernel_size, pad = ks / 2;
  const int H = 2 * p->reshape_width, W = p->reshape_height, HW = H * W, k = HW / 2, C1 = P * F;
  const int64_t Fw = (int64_t)C1 * HW;
  double *gent = grads[0], *grel = grads[1], *gw0 = grads[2], *gb0 = grads[3], *gfilt = grads[4], *gw1 = grads[5];
  double *gb1 = grads[6], *gfw = grads[7], *gfb = grads[8], *gw2 = grads[9], *gb2 = grads[10];
  double* img = (double*)malloc(sizeof(double) * (size_t)(B * P * HW));
  double* vin = (double*)malloc(sizeof(double) * (size_t)(B * P * HW));
  double* z1 = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* feat = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* hp = (double*)malloc(sizeof(double) * (size_t)(B * k));
  double* y2 = (double*)malloc(sizeof(double) * (size_t)(B * k));
  double* dh = (double*)malloc(sizeof(double) * (size_t)(B * k));
  double* dz = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* dv = (double*)malloc(sizeof(double) * (size_t)(B * P * HW));
  double* m0 = (double*)malloc(sizeof(double) * (size_t)P);
  double* i0 = (double*)malloc(sizeof(double) * (size_t)P);
  double* m1 = (double*)malloc(sizeof(double) * (size_t)C1);
  double* i1 = (double*)malloc(sizeof(double) * (size_t)C1);
  for (int64_t g0 = 0; g0 < Q; g0 += B) {
    /* forward */
    for (int64_t q = 0; q < B; ++q)
      for (int pp = 0; pp < P; ++pp)
        for (int i = 0; i < HW; ++i) {
          const int64_t c = p->perm[(int64_t)pp * HW + i];
          img[(q * P + pp) * HW + i] = c < k ? p->ent[e[g0 + q] * k + c] : p->rel[r[g0 + q] * k + (c - k)];
        }
    for (int pp = 0; pp < P; ++pp) {
      double s = 0.0, s2 = 0.0;
      for (int64_t q = 0; q < B; ++q) for (int i = 0; i < HW; ++i) s += img[(q * P + pp) * HW + i];
      m0[pp] = s / (double)(B * HW);
      for (int64_t q = 0; q < B; ++q)
        for (int i = 0; i < HW; ++i) { const double d = img[(q * P + pp) * HW + i] - m0[pp]; s2 += d * d; }
      i0[pp] = 1.0 / sqrt(s2 / (double)(B * HW) + p->bn0_eps);
    }
    for (int64_t q = 0; q < B; ++q)
      for (int pp = 0; pp < P; ++pp)
        for (int i = 0; i < HW; ++i) {
          const int64_t at = (q * P + pp) * HW + i;
          const double y = (img[at] - m0[pp]) * i0[pp] * p->bn0_weight[pp] + p->bn0_bias[pp];
          vin[at] = n0 ? y * n0[g0 * P * HW + at] : y;
        }
    for (int64_t q = 0; q < B; ++q)
      for (int pp = 0; pp < P; ++pp)
        for (int f = 0; f < F; ++f)
          for (int i = 0; i < H; ++i)
            for (int j = 0; j < W; ++j) {
              double acc = 0.0;
              for (int u = 0; u < ks; ++u)
                for (int vv = 0; vv < ks; ++vv)
                  acc += (double)p->conv_filt[((int64_t)f * ks + u) * ks + vv] *
                         vin[(q * P + pp) * HW + wrap(i + u - pad, H) * W + wrap(j + vv - pad, W)];
              z1[q * Fw + (int64_t)(pp * F + f) * HW + i * W + j] = acc;
            }
    for (int c = 0; c < C1; ++c) {
      double s = 0.0, s2 = 0.0;
      for (int64_t q = 0; q < B; ++q) for (int o = 0; o < HW; ++o) s += z1[q * Fw + (int64_t)c * HW + o];
      m1[c] = s / (double)(B * HW);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < HW; ++o) { const double d = z1[q * Fw + (int64_t)c * HW + o] - m1[c]; s2 += d * d; }
      i1[c] = 1.0 / sqrt(s2 / (double)(B * HW) + p->bn1_eps);
    }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t o = 0; o < Fw; ++o) {
        const int c = (int)(o / HW);
        const double y = (z1[q * Fw + o] - m1[c]) * i1[c] * p->bn1_weight[c] + p->bn1_bias[c];
        feat[q * Fw + o] = (y > 0 ? y : 0.0) * (n1 ? n1[(g0 + q) * C1 + c] : 1.0);
      }
    for (int64_t q = 0; q < B; ++q)
      for (int n = 0; n < k; ++n) {
        double acc = p->fc_bias[n];
        for (int64_t f = 0; f < Fw; ++f) acc += feat[q * Fw + f] * p->fc_weight[(int64_t)n * Fw + f];
        hp[q * k + n] = n2 ? acc * n2[(g0 + q) * k + n] : acc;
      }
    /* bn2, relu; backward of bn2 and the Linear layer */
    for (int j = 0; j < k; ++j) {
      double s = 0.0, s2 = 0.0;
      for (int64_t q = 0; q < B; ++q) s += hp[q * k + j];
      const double m2v = s / (double)B;
      for (int64_t q = 0; q < B; ++q) { const double d = hp[q * k + j] - m2v; s2 += d * d; }
      const double i2v = 1.0 / sqrt(s2 / (double)B + p->bn2_eps);
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q) {
        const double xh = (hp[q * k + j] - m2v) * i2v, y = xh * p->bn2_weight[j] + p->bn2_bias[j];
        y2[q * k + j] = y;
        if (x64) x64[(g0 + q) * k + j] = y > 0 ? y : 0.0;
        const double gy = y > 0 ? gx[(g0 + q) * k + j] : 0.0;
        sg += gy; sgx += gy * xh;
      }
      gw2[j] += sgx; gb2[j] += sg;
      for (int64_t q = 0; q < B; ++q) {
        const double xh = (hp[q * k + j] - m2v) * i2v;
        const double gy = y2[q * k + j] > 0 ? gx[(g0 + q) * k + j] : 0.0;
        double d = p->bn2_weight[j] * i2v * (gy - sg / (double)B - xh * sgx / (double)B);
        if (n2) d *= n2[(g0 + q) * k + j];
        dh[q * k + j] = d;
        gfb[j] += d;
      }
    }
    for (int n = 0; n < k; ++n)
      for (int64_t f = 0; f < Fw; ++f) {
        double acc = 0.0;
        for (int64_t q = 0; q < B; ++q) acc += dh[q * k + n] * feat[q * Fw + f];
        gfw[(int64_t)n * Fw + f] += acc;
      }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t f = 0; f < Fw; ++f) {
        double acc = 0.0;
        for (int n = 0; n < k; ++n) acc += dh[q * k + n] * p->fc_weight[(int64_t)n * Fw + f];
        dz[q * Fw + f] = acc;   /* d feat */
      }
    /* noise1, relu, bn1 backward -> dz1 */
    for (int c = 0; c < C1; ++c) {
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < HW; ++o) {
          const int64_t at = q * Fw + (int64_t)c * HW + o;
          const double xh = (z1[at] - m1[c]) * i1[c];
          const double y = xh * p->bn1_weight[c] + p->bn1_bias[c];
          const double g = y > 0 ? dz[at] * (n1 ? n1[(g0 + q) * C1 + c] : 1.0) : 0.0;
          dz[at] = g;
          sg += g; sgx += g * xh;
        }
      gw1[c] += sgx; gb1[c] += sg;
      const double nn = (double)(B * HW);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < HW; ++o) {
          const int64_t at = q * Fw + (int64_t)c * HW + o;
          const double xh = (z1[at] - m1[c]) * i1[c];
          dz[at] = p->bn1_weight[c] * i1[c] * (dz[at] - sg / nn - xh * sgx / nn);
        }
    }
    /* filter gradient (summed over the P images: the repeated filter bank) and the transposed circular conv */
    for (int64_t i = 0; i < B * P * HW; ++i) dv[i] = 0.0;
    for (int64_t q = 0; q < B; ++q)
      for (int pp = 0; pp < P; ++pp)
        for (int f = 0; f < F; ++f)
          for (int i = 0; i < H; ++i)
            for (int j = 0; j < W; ++j) {
              const double d = dz[q * Fw + (int64_t)(pp * F + f) * HW + i * W + j];
              for (int u = 0; u < ks; ++u)
                for (int vv = 0; vv < ks; ++vv) {
                  const int64_t src = (q * P + pp) * HW + wrap(i + u - pad, H) * W + wrap(j + vv - pad, W);
                  const int64_t t = ((int64_t)f * ks + u) * ks + vv;
                  gfilt[t] += d * vin[src];
                  dv[src] += d * p->conv_filt[t];
                }
            }
    /* noise0, bn0 backward per image, un-permute and scatter */
    for (int pp = 0; pp < P; ++pp) {
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q)
        for (int i = 0; i < HW; ++i) {
          const int64_t at = (q * P + pp) * HW + i;
          if (n0) dv[at] *= n0[g0 * P * HW + at];
          sg += dv[at]; sgx += dv[at] * (img[at] - m0[pp]) * i0[pp];
        }
      gw0[pp] += sgx; gb0[pp] += sg;
      const double nn = (double)(B * HW);
      for (int64_t q = 0; q < B; ++q)
        for (int i = 0; i < HW; ++i) {
          const int64_t at = (q * P + pp) * HW + i;
          const double xh = (img[at] - m0[pp]) * i0[pp];
          const double d = p->bn0_weight[pp] * i0[pp] * (dv[at] - sg / nn - xh * sgx / nn);
          const int64_t c = p->perm[(int64_t)pp * HW + i];
          if (c < k) gent[e[g0 + q] * k + c] += d;
          else grel[r[g0 + q] * k + (c - k)] += d;
        }
    }
  }
  free(img); free(vin); free(z1); free(feat); free(hp); free(y2); free(dh); free(dz); free(dv);
  free(m0); free(i0); free(m1); free(i1);
  return 0;
}
