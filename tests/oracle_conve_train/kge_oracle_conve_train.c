/* tests/oracle_conve_train/kge_oracle_conve_train.c — TEST INFRASTRUCTURE: CPU oracle of ConvE's training-mode trunk
 * (pykg2vec_b200/csrc/kge_conve_train.cuh, pykg2vec/models/projection.py:86-99 with self.training == True).
 *
 * kgeo_conve_train_fwd restates the kernels' canonical arithmetic (DESIGN.md §3, ConvE training) in scalar C with
 * explicit fmaf and no contraction (-ffp-contract=off): the CTA sum (256 per-thread chains, xor butterfly inside each
 * warp, warp sums in ascending order), the warp sum (32 lane chains, butterfly), the per-query partials combined in
 * ascending query order, the 9-tap conv chain, the Linear layer's 512-feature slices added in order, bn2's two passes.
 * x and the running statistics must equal the kernels' bit for bit.
 *
 * kgeo_conve_train_bwd64 is the same trunk in double, forward and backward (the analytic BatchNorm, conv and Linear
 * backward): the yardstick of the kernels' backward, whose float atomics and fp32 sums are checked against it within
 * the fp32 summation bound. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/kge_b200.h"

#define NT 256 /* CONVE_TR_THREADS */
#define CH 32

static float butterfly32(float* a) {
  for (int off = 16; off; off >>= 1) {
    float b[32];
    for (int l = 0; l < 32; ++l) b[l] = a[l] + a[l ^ off];
    memcpy(a, b, sizeof b);
  }
  return a[0];
}

/* CTA sum of the per-thread chains t[0..256): xor butterfly inside each warp, then the warp sums in ascending order */
static float cta_combine(float* t) {
  float s = butterfly32(t);
  for (int k = 1; k < NT / 32; ++k) s = s + butterfly32(t + 32 * k);
  return s;
}

/* CTA sum of v[0..n): thread t's fadd chain over t, t+256, ... from 0 */
static float cta_sum(const float* v, int n) {
  float t[NT];
  for (int i = 0; i < NT; ++i) t[i] = 0.0f;
  for (int i = 0; i < n; ++i) t[i % NT] = t[i % NT] + v[i];
  return cta_combine(t);
}

/* the CTA's centred sum of squares around m: fmaf(d, d, acc) chains of d = v - m */
static float cta_m2(const float* v, int n, float m) {
  float t[NT];
  for (int i = 0; i < NT; ++i) t[i] = 0.0f;
  for (int i = 0; i < n; ++i) { const float d = v[i] - m; t[i % NT] = fmaf(d, d, t[i % NT]); }
  return cta_combine(t);
}

/* warp sum of v[0..n) and the warp's centred sum of squares around s / n */
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

/* conve_tr_bn_stats_kernel for one channel c of C: st[g] = (mean, invstd), running statistics group after group */
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

int kgeo_conve_train_fwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                         const float* n0, const float* n1, const float* n2, float* x) {
  const int k = p->hidden_size, W = p->hidden_size_1, h2 = k / W, nimg = 2 * k;
  const int Ho = 2 * h2 - 2, Wo = W - 2, plane = Ho * Wo;
  const int64_t F = (int64_t)CH * plane, G = Q / B;
  float* img = (float*)malloc(sizeof(float) * (size_t)(Q * nimg));
  float* z1 = (float*)malloc(sizeof(float) * (size_t)(Q * F));
  float* hp = (float*)malloc(sizeof(float) * (size_t)(Q * k));
  float* part0 = (float*)malloc(sizeof(float) * (size_t)(Q * 2));
  float* part1 = (float*)malloc(sizeof(float) * (size_t)(Q * CH * 2));
  float* st0 = (float*)malloc(sizeof(float) * (size_t)(G * 2));
  float* st1 = (float*)malloc(sizeof(float) * (size_t)(G * CH * 2));
  float* xin = (float*)malloc(sizeof(float) * (size_t)nimg);
  float* feat = (float*)malloc(sizeof(float) * (size_t)F);
  for (int64_t q = 0; q < Q; ++q) {
    float* im = img + q * nimg;
    for (int i = 0; i < nimg; ++i) im[i] = i < k ? p->ent[e[q] * k + i] : p->rel[r[q] * k + (i - k)];
    const float s = cta_sum(im, nimg);
    part0[q * 2] = s;
    part0[q * 2 + 1] = cta_m2(im, nimg, s / (float)nimg);
  }
  bn_stats(part0, Q, B, 1, 0, (float)nimg, p->bn0_eps, p->bn0_momentum, st0, p->bn0_mean, p->bn0_var);
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    for (int i = 0; i < nimg; ++i) {
      float v = bn_apply(img[q * nimg + i], st0[g * 2], st0[g * 2 + 1], p->bn0_weight[0], p->bn0_bias[0]);
      xin[i] = n0 ? v * n0[q * nimg + i] : v;
    }
    float* zq = z1 + q * F;
    for (int c = 0; c < CH; ++c)
      for (int i = 0; i < Ho; ++i)
        for (int j = 0; j < Wo; ++j) {
          float acc = 0.0f;
          for (int di = 0; di < 3; ++di)
            for (int dj = 0; dj < 3; ++dj) acc = fmaf(p->conv_weight[c * 9 + di * 3 + dj], xin[(i + di) * W + j + dj], acc);
          zq[c * plane + i * Wo + j] = acc + p->conv_bias[c];
        }
    for (int c = 0; c < CH; ++c) warp_stats(zq + c * plane, plane, &part1[(q * CH + c) * 2], &part1[(q * CH + c) * 2 + 1]);
  }
  for (int c = 0; c < CH; ++c)
    bn_stats(part1, Q, B, CH, c, (float)plane, p->bn1_eps, p->bn1_momentum, st1, p->bn1_mean, p->bn1_var);
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    for (int64_t o = 0; o < F; ++o) {
      const int c = (int)(o / plane);
      float v = fmaxf(bn_apply(z1[q * F + o], st1[(g * CH + c) * 2], st1[(g * CH + c) * 2 + 1], p->bn1_weight[c],
                               p->bn1_bias[c]), 0.0f);
      feat[o] = n1 ? v * n1[q * CH + c] : v;
    }
    for (int n = 0; n < k; ++n) {   /* Linear: per-slice fmaf chains, slice sums added in order */
      const float* w = p->fc_weight + (int64_t)n * F;
      float total = 0.0f;
      for (int64_t f0 = 0; f0 < F; f0 += 512) {
        const int64_t f1 = f0 + 512 < F ? f0 + 512 : F;
        float acc = 0.0f;
        for (int64_t f = f0; f < f1; ++f) acc = fmaf(feat[f], w[f], acc);
        total = (f0 == 0) ? acc : total + acc;
      }
      total = total + p->fc_bias[n];
      hp[q * k + n] = n2 ? total * n2[q * k + n] : total;
    }
  }
  for (int j = 0; j < k; ++j) {   /* bn2: two passes per feature over each group's rows */
    const float nB = (float)B, w = p->bn2_weight[j], b = p->bn2_bias[j];
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
      for (int64_t i = g * B; i < (g + 1) * B; ++i) x[i * k + j] = fmaxf(bn_apply(hp[i * k + j], mean, invstd, w, b), 0.0f);
    }
  }
  free(img); free(z1); free(hp); free(part0); free(part1); free(st0); free(st1); free(xin); free(feat);
  return 0;
}

/* ---- fp64 forward + backward ------------------------------------------------------------------------------------ */

/* batch-norm statistics in double over the n values v[idx(i)] */
static void stats64(const double* v, int64_t n, int64_t stride, double* mean, double* invstd, double eps) {
  double s = 0.0, s2 = 0.0;
  for (int64_t i = 0; i < n; ++i) s += v[i * stride];
  const double m = s / (double)n;
  for (int64_t i = 0; i < n; ++i) { const double d = v[i * stride] - m; s2 += d * d; }
  *mean = m;
  *invstd = 1.0 / sqrt(s2 / (double)n + eps);
}

/* grads: 12 buffers in kge_conve_train_bwd order (ent, rel, bn0.w, bn0.b, conv.w, conv.b, bn1.w, bn1.b, fc.w, fc.b,
 * bn2.w, bn2.b), ACCUMULATED; gx [Q, k]; x64 (may be NULL) receives the fp64 forward's x */
int kgeo_conve_train_bwd64(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                           const float* n0, const float* n1, const float* n2, const double* gx, double* const* grads,
                           double* x64) {
  const int k = p->hidden_size, W = p->hidden_size_1, h2 = k / W, nimg = 2 * k;
  const int Ho = 2 * h2 - 2, Wo = W - 2, plane = Ho * Wo;
  const int64_t F = (int64_t)CH * plane;
  double *gent = grads[0], *grel = grads[1], *gw0 = grads[2], *gb0 = grads[3], *gcw = grads[4], *gcb = grads[5];
  double *gw1 = grads[6], *gb1 = grads[7], *gfw = grads[8], *gfb = grads[9], *gw2 = grads[10], *gb2 = grads[11];
  double* img = (double*)malloc(sizeof(double) * (size_t)(B * nimg));
  double* xin = (double*)malloc(sizeof(double) * (size_t)(B * nimg));
  double* z1 = (double*)malloc(sizeof(double) * (size_t)(B * F));
  double* feat = (double*)malloc(sizeof(double) * (size_t)(B * F));
  double* hp = (double*)malloc(sizeof(double) * (size_t)(B * k));
  double* y2 = (double*)malloc(sizeof(double) * (size_t)(B * k));
  double* dh = (double*)malloc(sizeof(double) * (size_t)(B * k));
  double* dz = (double*)malloc(sizeof(double) * (size_t)(B * F));
  double* dx = (double*)malloc(sizeof(double) * (size_t)(B * nimg));
  double m1[CH], i1[CH], m2v, i2v;
  for (int64_t g0 = 0; g0 < Q; g0 += B) {
    /* forward */
    for (int64_t q = 0; q < B; ++q)
      for (int i = 0; i < nimg; ++i)
        img[q * nimg + i] = i < k ? p->ent[e[g0 + q] * k + i] : p->rel[r[g0 + q] * k + (i - k)];
    double m0, i0;
    stats64(img, B * nimg, 1, &m0, &i0, p->bn0_eps);
    for (int64_t i = 0; i < B * nimg; ++i) {
      const double y = (img[i] - m0) * i0 * p->bn0_weight[0] + p->bn0_bias[0];
      xin[i] = n0 ? y * n0[g0 * nimg + i] : y;
    }
    for (int64_t q = 0; q < B; ++q)
      for (int c = 0; c < CH; ++c)
        for (int i = 0; i < Ho; ++i)
          for (int j = 0; j < Wo; ++j) {
            double acc = p->conv_bias[c];
            for (int di = 0; di < 3; ++di)
              for (int dj = 0; dj < 3; ++dj) acc += (double)p->conv_weight[c * 9 + di * 3 + dj] * xin[q * nimg + (i + di) * W + j + dj];
            z1[q * F + c * plane + i * Wo + j] = acc;
          }
    for (int c = 0; c < CH; ++c) {
      double s = 0.0, s2 = 0.0;
      for (int64_t q = 0; q < B; ++q) for (int o = 0; o < plane; ++o) s += z1[q * F + c * plane + o];
      m1[c] = s / (double)(B * plane);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < plane; ++o) { const double d = z1[q * F + c * plane + o] - m1[c]; s2 += d * d; }
      i1[c] = 1.0 / sqrt(s2 / (double)(B * plane) + p->bn1_eps);
    }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t o = 0; o < F; ++o) {
        const int c = (int)(o / plane);
        const double y = (z1[q * F + o] - m1[c]) * i1[c] * p->bn1_weight[c] + p->bn1_bias[c];
        feat[q * F + o] = (y > 0 ? y : 0.0) * (n1 ? n1[(g0 + q) * CH + c] : 1.0);
      }
    for (int64_t q = 0; q < B; ++q)
      for (int n = 0; n < k; ++n) {
        double acc = p->fc_bias[n];
        for (int64_t f = 0; f < F; ++f) acc += feat[q * F + f] * p->fc_weight[(int64_t)n * F + f];
        hp[q * k + n] = n2 ? acc * n2[(g0 + q) * k + n] : acc;
      }
    /* bn2, relu; backward of bn2 and the Linear layer, feature by feature */
    for (int j = 0; j < k; ++j) {
      stats64(hp + j, B, k, &m2v, &i2v, p->bn2_eps);
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
      for (int64_t f = 0; f < F; ++f) {
        double acc = 0.0;
        for (int64_t q = 0; q < B; ++q) acc += dh[q * k + n] * feat[q * F + f];
        gfw[(int64_t)n * F + f] += acc;
      }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t f = 0; f < F; ++f) {
        double acc = 0.0;
        for (int n = 0; n < k; ++n) acc += dh[q * k + n] * p->fc_weight[(int64_t)n * F + f];
        dz[q * F + f] = acc;   /* d feat */
      }
    /* relu mask, noise1, bn1 backward -> dz1 */
    for (int c = 0; c < CH; ++c) {
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < plane; ++o) {
          const int64_t at = q * F + c * plane + o;
          const double xh = (z1[at] - m1[c]) * i1[c], y = xh * p->bn1_weight[c] + p->bn1_bias[c];
          const double g = y > 0 ? dz[at] * (n1 ? n1[(g0 + q) * CH + c] : 1.0) : 0.0;
          dz[at] = g;
          sg += g; sgx += g * xh;
        }
      gw1[c] += sgx; gb1[c] += sg;
      const double nn = (double)(B * plane);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < plane; ++o) {
          const int64_t at = q * F + c * plane + o;
          const double xh = (z1[at] - m1[c]) * i1[c];
          dz[at] = p->bn1_weight[c] * i1[c] * (dz[at] - sg / nn - xh * sgx / nn);
          gcb[c] += dz[at];
        }
    }
    /* conv weight gradient and transposed conv */
    for (int64_t i = 0; i < B * nimg; ++i) dx[i] = 0.0;
    for (int64_t q = 0; q < B; ++q)
      for (int c = 0; c < CH; ++c)
        for (int i = 0; i < Ho; ++i)
          for (int j = 0; j < Wo; ++j) {
            const double d = dz[q * F + c * plane + i * Wo + j];
            for (int di = 0; di < 3; ++di)
              for (int dj = 0; dj < 3; ++dj) {
                const int at = (i + di) * W + j + dj;
                gcw[c * 9 + di * 3 + dj] += d * xin[q * nimg + at];
                dx[q * nimg + at] += d * p->conv_weight[c * 9 + di * 3 + dj];
              }
          }
    /* noise0, bn0 backward, scatter */
    double sg = 0.0, sgx = 0.0;
    for (int64_t i = 0; i < B * nimg; ++i) {
      if (n0) dx[i] *= n0[g0 * nimg + i];
      const double xh = (img[i] - m0) * i0;
      sg += dx[i]; sgx += dx[i] * xh;
    }
    gw0[0] += sgx; gb0[0] += sg;
    const double nn = (double)(B * nimg);
    for (int64_t q = 0; q < B; ++q)
      for (int i = 0; i < nimg; ++i) {
        const double xh = (img[q * nimg + i] - m0) * i0;
        const double d = p->bn0_weight[0] * i0 * (dx[q * nimg + i] - sg / nn - xh * sgx / nn);
        if (i < k) gent[e[g0 + q] * k + i] += d;
        else grel[r[g0 + q] * k + (i - k)] += d;
      }
  }
  free(img); free(xin); free(z1); free(feat); free(hp); free(y2); free(dh); free(dz); free(dx);
  return 0;
}
