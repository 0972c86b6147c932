/* tests/oracle_acre_train/kge_oracle_acre_train.c — TEST INFRASTRUCTURE: CPU oracle of AcrE's training-mode trunk
 * (pykg2vec_b200/csrc/kge_acre_train.cuh, pykg2vec/models/projection.py:706-734 with self.training == True).
 *
 * kgeo_acre_train_fwd restates the kernels' canonical arithmetic in scalar C with explicit fmaf and no contraction
 * (-ffp-contract=off): bn0's per-query partials as one CTA sum over the 400 stacked values (256 per-thread chains, xor
 * butterfly inside each warp, warp sums in ascending order), bn1's as warp sums per channel (32 lane chains,
 * butterfly), the partials combined in ascending query order; the convs as one fmaf chain from 0 in tap-major order
 * (tap (u, v) row-major, then the input channels), padding taps skipped, + bias as a separate add; the serial
 * residual a separate add; W_gate_e one fmaf chain over the 1600 gate inputs, + bias; the Linear layer's 512-feature
 * slices added in order; bn2's two passes.  x and the running statistics must equal the kernels' bit for bit.
 * Queries are independent within a phase, so the OpenMP loops do not change a bit.
 *
 * kgeo_acre_train_bwd64 is the same trunk in double, forward and backward (the analytic BatchNorm, dilated conv,
 * W_gate_e and Linear backward): the yardstick of the kernels' backward. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#include "../../include/kge_b200.h"

#define NT 256 /* CONVE_TR_THREADS */
#define PIX 400
#define SIDE 20
#define K 200

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

/* one dilated 3x3 conv Cin -> C over 20 x 20 maps (stride 400): tap-major fmaf chains, padding skipped, + bias */
static void conv_f32(const float* in, int Cin, int C, int d, const float* w, const float* bias, float* out) {
  for (int co = 0; co < C; ++co)
    for (int i = 0; i < SIDE; ++i)
      for (int j = 0; j < SIDE; ++j) {
        float acc = 0.0f;
        for (int u = 0; u < 3; ++u)
          for (int v = 0; v < 3; ++v) {
            const int ii = i + (u - 1) * d, jj = j + (v - 1) * d;
            if (ii < 0 || ii >= SIDE || jj < 0 || jj >= SIDE) continue;
            for (int ci = 0; ci < Cin; ++ci)
              acc = fmaf(w[(((int64_t)co * Cin + ci) * 3 + u) * 3 + v], in[ci * PIX + ii * SIDE + jj], acc);
          }
        out[co * PIX + i * SIDE + j] = bias ? acc + bias[co] : acc;
      }
}

static const float* conv_w(const kge_acre_train_t* p, int l) {
  return l == 0 ? p->conv1_weight : (l == 1 ? p->conv2_weight : p->conv3_weight);
}
static const float* conv_b(const kge_acre_train_t* p, int l) {
  return l == 0 ? p->conv1_bias : (l == 1 ? p->conv2_bias : p->conv3_bias);
}
static int dil(const kge_acre_train_t* p, int l) {
  return l == 0 ? p->first_atrous : (l == 1 ? p->second_atrous : p->third_atrous);
}

int kgeo_acre_train_fwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* n0, const float* n1, const float* n2, float* x) {
  const int C = p->in_channels, par = p->way == 1;
  const int64_t Fw = (int64_t)C * PIX, G = Q / B;
  float* img = (float*)malloc(sizeof(float) * (size_t)(Q * PIX));
  float* y = (float*)malloc(sizeof(float) * (size_t)(Q * Fw));
  float* hp = (float*)malloc(sizeof(float) * (size_t)(Q * K));
  float* part0 = (float*)malloc(sizeof(float) * (size_t)(Q * 2));
  float* part1 = (float*)malloc(sizeof(float) * (size_t)(Q * C * 2));
  float* st0 = (float*)malloc(sizeof(float) * (size_t)(G * 2));
  float* st1 = (float*)malloc(sizeof(float) * (size_t)(G * C * 2));
  for (int64_t q = 0; q < Q; ++q) {
    float* im = img + q * PIX;
    for (int i = 0; i < PIX; ++i) im[i] = i < K ? p->ent[e[q] * K + i] : p->rel[r[q] * K + (i - K)];
    const float s = cta_sum(im, PIX);
    part0[q * 2] = s;
    part0[q * 2 + 1] = cta_m2(im, PIX, s / (float)PIX);
  }
  bn_stats(part0, Q, B, 1, 0, (float)PIX, p->bn0_eps, p->bn0_momentum, st0, p->bn0_mean, p->bn0_var);
#pragma omp parallel for schedule(static)
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    float* v = (float*)malloc(sizeof(float) * PIX);
    float* m1 = (float*)malloc(sizeof(float) * (size_t)Fw);
    float* m2 = (float*)malloc(sizeof(float) * (size_t)Fw);
    float* m3 = (float*)malloc(sizeof(float) * (size_t)Fw);
    for (int i = 0; i < PIX; ++i) {
      const float t = bn_apply(img[q * PIX + i], st0[g * 2], st0[g * 2 + 1], p->bn0_weight[0], p->bn0_bias[0]);
      v[i] = n0 ? t * n0[q * PIX + i] : t;
    }
    float* yq = y + q * Fw;
    if (!par) {
      conv_f32(v, 1, C, dil(p, 0), conv_w(p, 0), conv_b(p, 0), m1);
      conv_f32(m1, C, C, dil(p, 1), conv_w(p, 1), conv_b(p, 1), m2);
      conv_f32(m2, C, C, dil(p, 2), conv_w(p, 2), conv_b(p, 2), m3);
      for (int64_t o = 0; o < Fw; ++o) yq[o] = m3[o] + v[o % PIX];
    } else {
      float gate[4 * PIX];
      conv_f32(v, 1, C, dil(p, 0), conv_w(p, 0), conv_b(p, 0), m1);
      conv_f32(v, 1, C, dil(p, 1), conv_w(p, 1), conv_b(p, 1), m2);
      conv_f32(v, 1, C, dil(p, 2), conv_w(p, 2), conv_b(p, 2), m3);
      for (int c = 0; c < C; ++c) {
        memcpy(gate, v, sizeof(float) * PIX);
        memcpy(gate + PIX, m1 + c * PIX, sizeof(float) * PIX);
        memcpy(gate + 2 * PIX, m2 + c * PIX, sizeof(float) * PIX);
        memcpy(gate + 3 * PIX, m3 + c * PIX, sizeof(float) * PIX);
        for (int n = 0; n < PIX; ++n) {   /* W_gate_e: one fmaf chain over the 1600 inputs, + bias */
          const float* wr = p->W_gate_e_weight + (int64_t)n * 4 * PIX;
          float acc = 0.0f;
          for (int t = 0; t < 4 * PIX; ++t) acc = fmaf(gate[t], wr[t], acc);
          yq[c * PIX + n] = acc + p->W_gate_e_bias[n];
        }
      }
    }
    for (int c = 0; c < C; ++c) warp_stats(yq + (int64_t)c * PIX, PIX, &part1[(q * C + c) * 2], &part1[(q * C + c) * 2 + 1]);
    free(v); free(m1); free(m2); free(m3);
  }
  for (int c = 0; c < C; ++c)
    bn_stats(part1, Q, B, C, c, (float)PIX, p->bn1_eps, p->bn1_momentum, st1, p->bn1_mean, p->bn1_var);
#pragma omp parallel for schedule(static)
  for (int64_t q = 0; q < Q; ++q) {
    const int64_t g = q / B;
    float* feat = (float*)malloc(sizeof(float) * (size_t)Fw);
    for (int64_t o = 0; o < Fw; ++o) {
      const int c = (int)(o / PIX);
      float t = bn_apply(y[q * Fw + o], st1[(g * C + c) * 2], st1[(g * C + c) * 2 + 1], p->bn1_weight[c],
                         p->bn1_bias[c]);
      t = fmaxf(t, 0.0f);
      feat[o] = n1 ? t * n1[q * C + c] : t;
    }
    for (int n = 0; n < K; ++n) {   /* Linear: per-slice fmaf chains, slice sums added in order */
      const float* fw = p->fc_weight + (int64_t)n * Fw;
      float total = 0.0f;
      for (int64_t f0 = 0; f0 < Fw; f0 += 512) {
        const int64_t f1 = f0 + 512 < Fw ? f0 + 512 : Fw;
        float acc = 0.0f;
        for (int64_t f = f0; f < f1; ++f) acc = fmaf(feat[f], fw[f], acc);
        total = (f0 == 0) ? acc : total + acc;
      }
      total = total + p->fc_bias[n];
      hp[q * K + n] = n2 ? total * n2[q * K + n] : total;
    }
    free(feat);
  }
  for (int j = 0; j < K; ++j) {   /* bn2: two passes per feature over each group's rows */
    const float nB = (float)B, wj = p->bn2_weight[j], bj = p->bn2_bias[j];
    for (int64_t g = 0; g < G; ++g) {
      float S = 0.0f;
      for (int64_t i = g * B; i < (g + 1) * B; ++i) S = S + hp[i * K + j];
      const float mean = S / nB;
      float M2 = 0.0f;
      for (int64_t i = g * B; i < (g + 1) * B; ++i) { const float d = hp[i * K + j] - mean; M2 = fmaf(d, d, M2); }
      const float var = M2 / nB, invstd = 1.0f / sqrtf(var + p->bn2_eps);
      if (p->bn2_mean) {
        p->bn2_mean[j] = fmaf(p->bn2_momentum, mean, (1.0f - p->bn2_momentum) * p->bn2_mean[j]);
        p->bn2_var[j] = fmaf(p->bn2_momentum, (var * nB) / (nB - 1.0f), (1.0f - p->bn2_momentum) * p->bn2_var[j]);
      }
      for (int64_t i = g * B; i < (g + 1) * B; ++i) x[i * K + j] = fmaxf(bn_apply(hp[i * K + j], mean, invstd, wj, bj), 0.0f);
    }
  }
  free(img); free(y); free(hp); free(part0); free(part1); free(st0); free(st1);
  return 0;
}

/* ---- fp64 forward + backward ------------------------------------------------------------------------------------ */

static void conv_f64(const double* in, int Cin, int C, int d, const float* w, const float* bias, double* out) {
  for (int co = 0; co < C; ++co)
    for (int i = 0; i < SIDE; ++i)
      for (int j = 0; j < SIDE; ++j) {
        double acc = bias ? bias[co] : 0.0;
        for (int u = 0; u < 3; ++u)
          for (int v = 0; v < 3; ++v) {
            const int ii = i + (u - 1) * d, jj = j + (v - 1) * d;
            if (ii < 0 || ii >= SIDE || jj < 0 || jj >= SIDE) continue;
            for (int ci = 0; ci < Cin; ++ci)
              acc += (double)w[(((int64_t)co * Cin + ci) * 3 + u) * 3 + v] * in[ci * PIX + ii * SIDE + jj];
          }
        out[co * PIX + i * SIDE + j] = acc;
      }
}

/* backward of conv_f64: gw / gb (may be NULL) += the weight / bias gradients, din (may be NULL) += d in */
static void conv_bwd64(const double* in, const double* dz, int Cin, int C, int d, const float* w, double* gw,
                       double* gb, double* din) {
  for (int co = 0; co < C; ++co)
    for (int i = 0; i < SIDE; ++i)
      for (int j = 0; j < SIDE; ++j) {
        const double g = dz[co * PIX + i * SIDE + j];
        if (gb) gb[co] += g;
        for (int u = 0; u < 3; ++u)
          for (int v = 0; v < 3; ++v) {
            const int ii = i + (u - 1) * d, jj = j + (v - 1) * d;
            if (ii < 0 || ii >= SIDE || jj < 0 || jj >= SIDE) continue;
            for (int ci = 0; ci < Cin; ++ci) {
              const int64_t t = (((int64_t)co * Cin + ci) * 3 + u) * 3 + v;
              gw[t] += g * in[ci * PIX + ii * SIDE + jj];
              if (din) din[ci * PIX + ii * SIDE + jj] += g * w[t];
            }
          }
      }
}

/* grads: 18 slots in kge_acre_train_bwd order (ent, rel, bn0.w, bn0.b, conv1.w, conv1.b, conv2.w, conv2.b, conv3.w,
 * conv3.b, W_gate_e.w, W_gate_e.b, bn1.w, bn1.b, fc.w, fc.b, bn2.w, bn2.b), ACCUMULATED; absent parameters' slots
 * NULL; gx [Q, 200]; x64 (may be NULL) receives the fp64 forward's x */
int kgeo_acre_train_bwd64(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                          const float* n0, const float* n1, const float* n2, const double* gx, double* const* grads,
                          double* x64) {
  const int C = p->in_channels, par = p->way == 1;
  const int64_t Fw = (int64_t)C * PIX;
  double *gent = grads[0], *grel = grads[1], *gw0 = grads[2], *gb0 = grads[3], *ggw = grads[10], *ggb = grads[11];
  double *gw1 = grads[12], *gb1 = grads[13], *gfw = grads[14], *gfb = grads[15], *gw2 = grads[16], *gb2 = grads[17];
  double* img = (double*)malloc(sizeof(double) * (size_t)(B * PIX));
  double* vin = (double*)malloc(sizeof(double) * (size_t)(B * PIX));
  double* m1 = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* m2 = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* m3 = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* y = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* feat = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* hp = (double*)malloc(sizeof(double) * (size_t)(B * K));
  double* y2 = (double*)malloc(sizeof(double) * (size_t)(B * K));
  double* dh = (double*)malloc(sizeof(double) * (size_t)(B * K));
  double* dy = (double*)malloc(sizeof(double) * (size_t)(B * Fw));
  double* d2 = (double*)malloc(sizeof(double) * (size_t)Fw);
  double* d1 = (double*)malloc(sizeof(double) * (size_t)Fw);
  double* dv = (double*)malloc(sizeof(double) * (size_t)(B * PIX));
  double* m1s = (double*)malloc(sizeof(double) * (size_t)C);
  double* i1s = (double*)malloc(sizeof(double) * (size_t)C);
  double gate[4 * PIX], dgate[4 * PIX];
  for (int64_t g0 = 0; g0 < Q; g0 += B) {
    /* forward */
    double s = 0.0, s2 = 0.0;
    for (int64_t q = 0; q < B; ++q)
      for (int i = 0; i < PIX; ++i) {
        img[q * PIX + i] = i < K ? p->ent[e[g0 + q] * K + i] : p->rel[r[g0 + q] * K + (i - K)];
        s += img[q * PIX + i];
      }
    const double m0 = s / (double)(B * PIX);
    for (int64_t i = 0; i < B * PIX; ++i) s2 += (img[i] - m0) * (img[i] - m0);
    const double i0 = 1.0 / sqrt(s2 / (double)(B * PIX) + p->bn0_eps);
    for (int64_t i = 0; i < B * PIX; ++i) {
      const double t = (img[i] - m0) * i0 * p->bn0_weight[0] + p->bn0_bias[0];
      vin[i] = n0 ? t * n0[g0 * PIX + i] : t;
    }
    for (int64_t q = 0; q < B; ++q) {
      const double* v = vin + q * PIX;
      double* yq = y + q * Fw;
      if (!par) {
        conv_f64(v, 1, C, dil(p, 0), conv_w(p, 0), conv_b(p, 0), m1 + q * Fw);
        conv_f64(m1 + q * Fw, C, C, dil(p, 1), conv_w(p, 1), conv_b(p, 1), m2 + q * Fw);
        conv_f64(m2 + q * Fw, C, C, dil(p, 2), conv_w(p, 2), conv_b(p, 2), m3 + q * Fw);
        for (int64_t o = 0; o < Fw; ++o) yq[o] = m3[q * Fw + o] + v[o % PIX];
      } else {
        for (int l = 0; l < 3; ++l)
          conv_f64(v, 1, C, dil(p, l), conv_w(p, l), conv_b(p, l), (l == 0 ? m1 : (l == 1 ? m2 : m3)) + q * Fw);
        for (int c = 0; c < C; ++c) {
          memcpy(gate, v, sizeof(double) * PIX);
          memcpy(gate + PIX, m1 + q * Fw + c * PIX, sizeof(double) * PIX);
          memcpy(gate + 2 * PIX, m2 + q * Fw + c * PIX, sizeof(double) * PIX);
          memcpy(gate + 3 * PIX, m3 + q * Fw + c * PIX, sizeof(double) * PIX);
          for (int n = 0; n < PIX; ++n) {
            double acc = p->W_gate_e_bias[n];
            for (int t = 0; t < 4 * PIX; ++t) acc += gate[t] * p->W_gate_e_weight[(int64_t)n * 4 * PIX + t];
            yq[c * PIX + n] = acc;
          }
        }
      }
    }
    for (int c = 0; c < C; ++c) {
      double sc = 0.0, sc2 = 0.0;
      for (int64_t q = 0; q < B; ++q) for (int o = 0; o < PIX; ++o) sc += y[q * Fw + c * PIX + o];
      m1s[c] = sc / (double)(B * PIX);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < PIX; ++o) { const double d = y[q * Fw + c * PIX + o] - m1s[c]; sc2 += d * d; }
      i1s[c] = 1.0 / sqrt(sc2 / (double)(B * PIX) + p->bn1_eps);
    }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t o = 0; o < Fw; ++o) {
        const int c = (int)(o / PIX);
        const double t = (y[q * Fw + o] - m1s[c]) * i1s[c] * p->bn1_weight[c] + p->bn1_bias[c];
        feat[q * Fw + o] = (t > 0 ? t : 0.0) * (n1 ? n1[(g0 + q) * C + c] : 1.0);
      }
    for (int64_t q = 0; q < B; ++q)
      for (int n = 0; n < K; ++n) {
        double acc = p->fc_bias[n];
        for (int64_t f = 0; f < Fw; ++f) acc += feat[q * Fw + f] * p->fc_weight[(int64_t)n * Fw + f];
        hp[q * K + n] = n2 ? acc * n2[(g0 + q) * K + n] : acc;
      }
    /* bn2, relu; backward of bn2 and the Linear layer */
    for (int j = 0; j < K; ++j) {
      double sj = 0.0, sj2 = 0.0;
      for (int64_t q = 0; q < B; ++q) sj += hp[q * K + j];
      const double mj = sj / (double)B;
      for (int64_t q = 0; q < B; ++q) { const double d = hp[q * K + j] - mj; sj2 += d * d; }
      const double ij = 1.0 / sqrt(sj2 / (double)B + p->bn2_eps);
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q) {
        const double xh = (hp[q * K + j] - mj) * ij, t = xh * p->bn2_weight[j] + p->bn2_bias[j];
        y2[q * K + j] = t;
        if (x64) x64[(g0 + q) * K + j] = t > 0 ? t : 0.0;
        const double gy = t > 0 ? gx[(g0 + q) * K + j] : 0.0;
        sg += gy; sgx += gy * xh;
      }
      gw2[j] += sgx; gb2[j] += sg;
      for (int64_t q = 0; q < B; ++q) {
        const double xh = (hp[q * K + j] - mj) * ij;
        const double gy = y2[q * K + j] > 0 ? gx[(g0 + q) * K + j] : 0.0;
        double d = p->bn2_weight[j] * ij * (gy - sg / (double)B - xh * sgx / (double)B);
        if (n2) d *= n2[(g0 + q) * K + j];
        dh[q * K + j] = d;
        gfb[j] += d;
      }
    }
    for (int n = 0; n < K; ++n)
      for (int64_t f = 0; f < Fw; ++f) {
        double acc = 0.0;
        for (int64_t q = 0; q < B; ++q) acc += dh[q * K + n] * feat[q * Fw + f];
        gfw[(int64_t)n * Fw + f] += acc;
      }
    for (int64_t q = 0; q < B; ++q)
      for (int64_t f = 0; f < Fw; ++f) {
        double acc = 0.0;
        for (int n = 0; n < K; ++n) acc += dh[q * K + n] * p->fc_weight[(int64_t)n * Fw + f];
        dy[q * Fw + f] = acc;   /* d feat */
      }
    /* noise1, relu, bn1 backward -> dy */
    for (int c = 0; c < C; ++c) {
      double sg = 0.0, sgx = 0.0;
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < PIX; ++o) {
          const int64_t at = q * Fw + (int64_t)c * PIX + o;
          const double xh = (y[at] - m1s[c]) * i1s[c];
          const double t = xh * p->bn1_weight[c] + p->bn1_bias[c];
          const double g = t > 0 ? dy[at] * (n1 ? n1[(g0 + q) * C + c] : 1.0) : 0.0;
          dy[at] = g;
          sg += g; sgx += g * xh;
        }
      gw1[c] += sgx; gb1[c] += sg;
      const double nn = (double)(B * PIX);
      for (int64_t q = 0; q < B; ++q)
        for (int o = 0; o < PIX; ++o) {
          const int64_t at = q * Fw + (int64_t)c * PIX + o;
          const double xh = (y[at] - m1s[c]) * i1s[c];
          dy[at] = p->bn1_weight[c] * i1s[c] * (dy[at] - sg / nn - xh * sgx / nn);
        }
    }
    /* the convs' backward -> d v */
    for (int64_t i = 0; i < B * PIX; ++i) dv[i] = 0.0;
    for (int64_t q = 0; q < B; ++q) {
      const double* dyq = dy + q * Fw;
      double* dvq = dv + q * PIX;
      if (!par) {
        for (int64_t o = 0; o < Fw; ++o) dvq[o % PIX] += dyq[o];   /* the residual */
        memset(d2, 0, sizeof(double) * (size_t)Fw);
        memset(d1, 0, sizeof(double) * (size_t)Fw);
        conv_bwd64(m2 + q * Fw, dyq, C, C, dil(p, 2), conv_w(p, 2), grads[8], grads[9], d2);
        conv_bwd64(m1 + q * Fw, d2, C, C, dil(p, 1), conv_w(p, 1), grads[6], grads[7], d1);
        conv_bwd64(vin + q * PIX, d1, 1, C, dil(p, 0), conv_w(p, 0), grads[4], grads[5], dvq);
      } else {
        double* dz[3] = {m1 + q * Fw, m2 + q * Fw, m3 + q * Fw};   /* reused as the convs' output gradients */
        for (int c = 0; c < C; ++c) {
          memcpy(gate, vin + q * PIX, sizeof(double) * PIX);
          memcpy(gate + PIX, dz[0] + c * PIX, sizeof(double) * PIX);
          memcpy(gate + 2 * PIX, dz[1] + c * PIX, sizeof(double) * PIX);
          memcpy(gate + 3 * PIX, dz[2] + c * PIX, sizeof(double) * PIX);
          for (int t = 0; t < 4 * PIX; ++t) dgate[t] = 0.0;
          for (int n = 0; n < PIX; ++n) {
            const double g = dyq[c * PIX + n];
            ggb[n] += g;
            const float* wr = p->W_gate_e_weight + (int64_t)n * 4 * PIX;
            for (int t = 0; t < 4 * PIX; ++t) {
              ggw[(int64_t)n * 4 * PIX + t] += g * gate[t];
              dgate[t] += g * wr[t];
            }
          }
          for (int i = 0; i < PIX; ++i) dvq[i] += dgate[i];
          for (int l = 0; l < 3; ++l) memcpy(dz[l] + c * PIX, dgate + (l + 1) * PIX, sizeof(double) * PIX);
        }
        for (int l = 0; l < 3; ++l)
          conv_bwd64(vin + q * PIX, dz[l], 1, C, dil(p, l), conv_w(p, l), grads[4 + 2 * l], grads[5 + 2 * l], dvq);
      }
    }
    /* noise0, bn0 backward, scatter */
    double sg = 0.0, sgx = 0.0;
    for (int64_t i = 0; i < B * PIX; ++i) {
      if (n0) dv[i] *= n0[g0 * PIX + i];
      sg += dv[i]; sgx += dv[i] * (img[i] - m0) * i0;
    }
    gw0[0] += sgx; gb0[0] += sg;
    const double nn = (double)(B * PIX);
    for (int64_t q = 0; q < B; ++q)
      for (int i = 0; i < PIX; ++i) {
        const int64_t at = q * PIX + i;
        const double d = p->bn0_weight[0] * i0 * (dv[at] - sg / nn - (img[at] - m0) * i0 * sgx / nn);
        if (i < K) gent[e[g0 + q] * K + i] += d;
        else grel[r[g0 + q] * K + (i - K)] += d;
      }
  }
  free(img); free(vin); free(m1); free(m2); free(m3); free(y); free(feat); free(hp); free(y2); free(dh); free(dy);
  free(d2); free(d1); free(dv); free(m1s); free(i1s);
  return 0;
}
