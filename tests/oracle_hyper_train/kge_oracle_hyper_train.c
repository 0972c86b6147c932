/* tests/oracle_hyper_train/kge_oracle_hyper_train.c — TEST INFRASTRUCTURE: CPU oracle of HypER's training-mode trunk
 * (pykg2vec_b200/csrc/kge_hyper_train.cuh, pykg2vec/models/projection.py:581-606 with self.training == True).
 *
 * kgeo_hyper_train_fwd restates the kernels' canonical arithmetic in scalar C with explicit fmaf and no contraction
 * (-ffp-contract=off): the filters as one fmaf chain over dr then + fc1.bias, the CTA sum (256 per-thread chains, xor
 * butterfly inside each warp, warp sums in ascending order), the warp sum (32 lane chains, butterfly), the per-query
 * partials combined in ascending query order, the 9-tap conv chain, the Linear layer's 512-feature slices added in
 * order, bn2's two passes.  x and the running statistics must equal the kernels' bit for bit.
 *
 * kgeo_hyper_train_bwd64 is the same trunk in double, forward and backward (the analytic BatchNorm, conv, Linear and
 * filter-generator backward, the embeddings' padding rows skipped): the yardstick of the kernels' backward. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/kge_b200.h"

#define NT 256 /* CONVE_TR_THREADS */
#define CH 32
#define FW 9
#define NF 288

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

static void filters(const kge_hyper_train_t* p, int64_t rr, float* w) {
  const int dr = p->rel_hidden_size;
  const float* rv = p->rel + rr * dr;
  for (int o = 0; o < NF; ++o) {
    const float* fw = p->fc1_weight + (int64_t)o * dr;
    float acc = 0.0f;
    for (int i = 0; i < dr; ++i) acc = fmaf(rv[i], fw[i], acc);
    w[o] = acc + p->fc1_bias[o];
  }
}

int kgeo_hyper_train_fwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                         const float* n0, const float* n1, const float* n2, float* x) {
  const int de = p->ent_hidden_size, Wo = de - 8;
  const int64_t F = (int64_t)CH * Wo, G = Q / B;
  float* img = (float*)malloc(sizeof(float) * (size_t)(Q * de));
  float* z1 = (float*)malloc(sizeof(float) * (size_t)(Q * F));
  float* hp = (float*)malloc(sizeof(float) * (size_t)(Q * de));
  float* part0 = (float*)malloc(sizeof(float) * (size_t)(Q * 2));
  float* part1 = (float*)malloc(sizeof(float) * (size_t)(Q * CH * 2));
  float* st0 = (float*)malloc(sizeof(float) * (size_t)(G * 2));
  float* st1 = (float*)malloc(sizeof(float) * (size_t)(G * CH * 2));
  float* v = (float*)malloc(sizeof(float) * (size_t)de);
  float* feat = (float*)malloc(sizeof(float) * (size_t)F);
  float w[NF];
  for (int64_t q = 0; q < Q; ++q) {
    float* im = img + q * de;
    for (int i = 0; i < de; ++i) im[i] = p->ent[e[q] * de + i];
    const float s = cta_sum(im, de);
    part0[q * 2] = s;
    part0[q * 2 + 1] = cta_m2(im, de, s / (float)de);
  }
  bn_stats(part0, Q, B, 1, 0, (float)de, p->bn0_eps, p->bn0_momentum, st0, p->bn0_mean, p->bn0_var);
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    for (int i = 0; i < de; ++i) {
      const float y = bn_apply(img[q * de + i], st0[g * 2], st0[g * 2 + 1], p->bn0_weight[0], p->bn0_bias[0]);
      v[i] = n0 ? y * n0[q * de + i] : y;
    }
    filters(p, r[q], w);
    float* zq = z1 + q * F;
    for (int c = 0; c < CH; ++c)
      for (int j = 0; j < Wo; ++j) {
        float acc = 0.0f;
        for (int t = 0; t < FW; ++t) acc = fmaf(w[c * FW + t], v[j + t], acc);
        zq[c * Wo + j] = acc;
      }
    for (int c = 0; c < CH; ++c) warp_stats(zq + c * Wo, Wo, &part1[(q * CH + c) * 2], &part1[(q * CH + c) * 2 + 1]);
  }
  for (int c = 0; c < CH; ++c)
    bn_stats(part1, Q, B, CH, c, (float)Wo, p->bn1_eps, p->bn1_momentum, st1, p->bn1_mean, p->bn1_var);
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    for (int64_t o = 0; o < F; ++o) {
      const int c = (int)(o / Wo);
      const float y = bn_apply(z1[q * F + o], st1[(g * CH + c) * 2], st1[(g * CH + c) * 2 + 1], p->bn1_weight[c],
                               p->bn1_bias[c]);
      feat[o] = n1 ? y * n1[q * CH + c] : y;
    }
    for (int n = 0; n < de; ++n) {   /* Linear: per-slice fmaf chains, slice sums added in order */
      const float* fw = p->fc_weight + (int64_t)n * F;
      float total = 0.0f;
      for (int64_t f0 = 0; f0 < F; f0 += 512) {
        const int64_t f1 = f0 + 512 < F ? f0 + 512 : F;
        float acc = 0.0f;
        for (int64_t f = f0; f < f1; ++f) acc = fmaf(feat[f], fw[f], acc);
        total = (f0 == 0) ? acc : total + acc;
      }
      total = total + p->fc_bias[n];
      hp[q * de + n] = n2 ? total * n2[q * de + n] : total;
    }
  }
  for (int j = 0; j < de; ++j) {   /* bn2: two passes per feature over each group's rows */
    const float nB = (float)B, wj = p->bn2_weight[j], bj = p->bn2_bias[j];
    for (int64_t g = 0; g < G; ++g) {
      float S = 0.0f;
      for (int64_t i = g * B; i < (g + 1) * B; ++i) S = S + hp[i * de + j];
      const float mean = S / nB;
      float M2 = 0.0f;
      for (int64_t i = g * B; i < (g + 1) * B; ++i) { const float d = hp[i * de + j] - mean; M2 = fmaf(d, d, M2); }
      const float var = M2 / nB, invstd = 1.0f / sqrtf(var + p->bn2_eps);
      if (p->bn2_mean) {
        p->bn2_mean[j] = fmaf(p->bn2_momentum, mean, (1.0f - p->bn2_momentum) * p->bn2_mean[j]);
        p->bn2_var[j] = fmaf(p->bn2_momentum, (var * nB) / (nB - 1.0f), (1.0f - p->bn2_momentum) * p->bn2_var[j]);
      }
      for (int64_t i = g * B; i < (g + 1) * B; ++i) x[i * de + j] = fmaxf(bn_apply(hp[i * de + j], mean, invstd, wj, bj), 0.0f);
    }
  }
  free(img); free(z1); free(hp); free(part0); free(part1); free(st0); free(st1); free(v); free(feat);
  return 0;
}

/* ---- fp64 forward + backward ------------------------------------------------------------------------------------ */

static void stats64(const double* v, int64_t n, int64_t stride, double* mean, double* invstd, double eps) {
  double s = 0.0, s2 = 0.0;
  for (int64_t i = 0; i < n; ++i) s += v[i * stride];
  const double m = s / (double)n;
  for (int64_t i = 0; i < n; ++i) { const double d = v[i * stride] - m; s2 += d * d; }
  *mean = m;
  *invstd = 1.0 / sqrt(s2 / (double)n + eps);
}

/* grads: 12 buffers in kge_hyper_train_bwd order (ent, rel, bn0.w, bn0.b, bn1.w, bn1.b, fc.w, fc.b, bn2.w, bn2.b,
 * fc1.w, fc1.b), ACCUMULATED; gx [Q, de]; x64 (may be NULL) receives the fp64 forward's x */
int kgeo_hyper_train_bwd64(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                           const float* n0, const float* n1, const float* n2, const double* gx, double* const* grads,
                           double* x64) {
  const int de = p->ent_hidden_size, dr = p->rel_hidden_size, Wo = de - 8;
  const int64_t F = (int64_t)CH * Wo;
  double *gent = grads[0], *grel = grads[1], *gw0 = grads[2], *gb0 = grads[3], *gw1 = grads[4], *gb1 = grads[5];
  double *gfw = grads[6], *gfb = grads[7], *gw2 = grads[8], *gb2 = grads[9], *gf1w = grads[10], *gf1b = grads[11];
  double* img = (double*)malloc(sizeof(double) * (size_t)(B * de));
  double* xin = (double*)malloc(sizeof(double) * (size_t)(B * de));
  double* wq = (double*)malloc(sizeof(double) * (size_t)(B * NF));
  double* z1 = (double*)malloc(sizeof(double) * (size_t)(B * F));
  double* feat = (double*)malloc(sizeof(double) * (size_t)(B * F));
  double* hp = (double*)malloc(sizeof(double) * (size_t)(B * de));
  double* y2 = (double*)malloc(sizeof(double) * (size_t)(B * de));
  double* dh = (double*)malloc(sizeof(double) * (size_t)(B * de));
  double* dz = (double*)malloc(sizeof(double) * (size_t)(B * F));
  double* dx = (double*)malloc(sizeof(double) * (size_t)(B * de));
  double* dw = (double*)malloc(sizeof(double) * (size_t)(B * NF));
  double m1[CH], i1[CH], m2v, i2v;
  for (int64_t g0 = 0; g0 < Q; g0 += B) {
    /* forward */
    for (int64_t q = 0; q < B; ++q) {
      for (int i = 0; i < de; ++i) img[q * de + i] = p->ent[e[g0 + q] * de + i];
      for (int o = 0; o < NF; ++o) {
        double acc = p->fc1_bias[o];
        for (int i = 0; i < dr; ++i) acc += (double)p->rel[r[g0 + q] * dr + i] * p->fc1_weight[(int64_t)o * dr + i];
        wq[q * NF + o] = acc;
      }
    }
    double m0, i0;
    stats64(img, B * de, 1, &m0, &i0, p->bn0_eps);
    for (int64_t i = 0; i < B * de; ++i) {
      const double y = (img[i] - m0) * i0 * p->bn0_weight[0] + p->bn0_bias[0];
      xin[i] = n0 ? y * n0[g0 * de + i] : y;
    }
    for (int64_t q = 0; q < B; ++q)
      for (int c = 0; c < CH; ++c)
        for (int j = 0; j < Wo; ++j) {
          double acc = 0.0;
          for (int t = 0; t < FW; ++t) acc += wq[q * NF + c * FW + t] * xin[q * de + j + t];
          z1[q * F + c * Wo + j] = acc;
        }
    for (int c = 0; c < CH; ++c) {
      double s = 0.0, s2 = 0.0;
      for (int64_t q = 0; q < B; ++q) for (int o = 0; o < Wo; ++o) s += z1[q * F + c * Wo + o];
      m1[c] = s / (double)(B * Wo);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < Wo; ++o) { const double d = z1[q * F + c * Wo + o] - m1[c]; s2 += d * d; }
      i1[c] = 1.0 / sqrt(s2 / (double)(B * Wo) + p->bn1_eps);
    }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t o = 0; o < F; ++o) {
        const int c = (int)(o / Wo);
        const double y = (z1[q * F + o] - m1[c]) * i1[c] * p->bn1_weight[c] + p->bn1_bias[c];
        feat[q * F + o] = y * (n1 ? n1[(g0 + q) * CH + c] : 1.0);
      }
    for (int64_t q = 0; q < B; ++q)
      for (int n = 0; n < de; ++n) {
        double acc = p->fc_bias[n];
        for (int64_t f = 0; f < F; ++f) acc += feat[q * F + f] * p->fc_weight[(int64_t)n * F + f];
        hp[q * de + n] = n2 ? acc * n2[(g0 + q) * de + n] : acc;
      }
    /* bn2, relu; backward of bn2 and the Linear layer */
    for (int j = 0; j < de; ++j) {
      stats64(hp + j, B, de, &m2v, &i2v, p->bn2_eps);
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q) {
        const double xh = (hp[q * de + j] - m2v) * i2v, y = xh * p->bn2_weight[j] + p->bn2_bias[j];
        y2[q * de + j] = y;
        if (x64) x64[(g0 + q) * de + j] = y > 0 ? y : 0.0;
        const double gy = y > 0 ? gx[(g0 + q) * de + j] : 0.0;
        sg += gy; sgx += gy * xh;
      }
      gw2[j] += sgx; gb2[j] += sg;
      for (int64_t q = 0; q < B; ++q) {
        const double xh = (hp[q * de + j] - m2v) * i2v;
        const double gy = y2[q * de + j] > 0 ? gx[(g0 + q) * de + j] : 0.0;
        double d = p->bn2_weight[j] * i2v * (gy - sg / (double)B - xh * sgx / (double)B);
        if (n2) d *= n2[(g0 + q) * de + j];
        dh[q * de + j] = d;
        gfb[j] += d;
      }
    }
    for (int n = 0; n < de; ++n)
      for (int64_t f = 0; f < F; ++f) {
        double acc = 0.0;
        for (int64_t q = 0; q < B; ++q) acc += dh[q * de + n] * feat[q * F + f];
        gfw[(int64_t)n * F + f] += acc;
      }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t f = 0; f < F; ++f) {
        double acc = 0.0;
        for (int n = 0; n < de; ++n) acc += dh[q * de + n] * p->fc_weight[(int64_t)n * F + f];
        dz[q * F + f] = acc;   /* d feat */
      }
    /* noise1, bn1 backward (no ReLU) -> dz1 */
    for (int c = 0; c < CH; ++c) {
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < Wo; ++o) {
          const int64_t at = q * F + c * Wo + o;
          const double xh = (z1[at] - m1[c]) * i1[c];
          const double g = dz[at] * (n1 ? n1[(g0 + q) * CH + c] : 1.0);
          dz[at] = g;
          sg += g; sgx += g * xh;
        }
      gw1[c] += sgx; gb1[c] += sg;
      const double nn = (double)(B * Wo);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < Wo; ++o) {
          const int64_t at = q * F + c * Wo + o;
          const double xh = (z1[at] - m1[c]) * i1[c];
          dz[at] = p->bn1_weight[c] * i1[c] * (dz[at] - sg / nn - xh * sgx / nn);
        }
    }
    /* filter gradient and transposed filter */
    for (int64_t i = 0; i < B * de; ++i) dx[i] = 0.0;
    for (int64_t i = 0; i < B * NF; ++i) dw[i] = 0.0;
    for (int64_t q = 0; q < B; ++q)
      for (int c = 0; c < CH; ++c)
        for (int j = 0; j < Wo; ++j) {
          const double d = dz[q * F + c * Wo + j];
          for (int t = 0; t < FW; ++t) {
            dw[q * NF + c * FW + t] += d * xin[q * de + j + t];
            dx[q * de + j + t] += d * wq[q * NF + c * FW + t];
          }
        }
    /* the filter generator fc1 and the relation rows */
    for (int64_t q = 0; q < B; ++q) {
      const int64_t rr = r[g0 + q];
      for (int o = 0; o < NF; ++o) {
        const double d = dw[q * NF + o];
        gf1b[o] += d;
        for (int i = 0; i < dr; ++i) {
          gf1w[(int64_t)o * dr + i] += d * p->rel[rr * dr + i];
          if (rr != p->rel_padding_idx) grel[rr * dr + i] += d * p->fc1_weight[(int64_t)o * dr + i];
        }
      }
    }
    /* noise0, bn0 backward, scatter */
    double sg = 0.0, sgx = 0.0;
    for (int64_t i = 0; i < B * de; ++i) {
      if (n0) dx[i] *= n0[g0 * de + i];
      const double xh = (img[i] - m0) * i0;
      sg += dx[i]; sgx += dx[i] * xh;
    }
    gw0[0] += sgx; gb0[0] += sg;
    const double nn = (double)(B * de);
    for (int64_t q = 0; q < B; ++q) {
      if (e[g0 + q] == p->ent_padding_idx) continue;
      for (int i = 0; i < de; ++i) {
        const double xh = (img[q * de + i] - m0) * i0;
        gent[e[g0 + q] * de + i] += p->bn0_weight[0] * i0 * (dx[q * de + i] - sg / nn - xh * sgx / nn);
      }
    }
  }
  free(img); free(xin); free(wq); free(z1); free(feat); free(hp); free(y2); free(dh); free(dz); free(dx); free(dw);
  return 0;
}
