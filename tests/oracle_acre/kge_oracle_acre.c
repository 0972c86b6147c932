/* tests/oracle_acre/kge_oracle_acre.c — TEST INFRASTRUCTURE: scalar C restatement of AcrE's inference trunk in
 * the canonical arithmetic of pykg2vec_b200/csrc/kge_acre.cuh (the CUDA path must agree with it bit for bit).
 * Built with gcc -O2 -ffp-contract=off -fno-fast-math -fopenmp -mfma (fmaf() is explicit, nothing else is
 * contracted) by tests/acre_util.py; the projection tail and its rank counts stay with oracle/.  Nothing in
 * pykg2vec_b200/ can reach it. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* BatchNorm in inference mode folded to fmaf(v, a, c), as ATen folds it (same rule as oracle/kge_oracle.c) */
static void bn_fold(float w, float b, float mean, float var, float eps, float* a, float* c) {
  *a = w / sqrtf(var + eps);
  *c = b - mean * *a;
}

typedef struct kge_acre {
  int32_t in_channels, way, first_atrous, second_atrous, third_atrous, hidden_size;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* conv1_weight; const float* conv1_bias;
  const float* conv2_weight; const float* conv2_bias;
  const float* conv3_weight; const float* conv3_bias;
  const float* W_gate_e_weight; const float* W_gate_e_bias;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias; const float* bn2_mean; const float* bn2_var;
} kge_acre_t;

/* one dilated 3x3 conv, Cin -> C channels on 20 x 20 maps: per output (co, i, j) one fmaf chain from 0 over the
 * taps (u, v) row-major and, within a tap, the input channels in order; taps in the zero padding are skipped;
 * then + bias (if any) as a separate add */
static void conv(const float* in, int Cin, int C, int d, const float* w, const float* bias, float* out) {
  for (int co = 0; co < C; ++co)
    for (int i = 0; i < 20; ++i)
      for (int j = 0; j < 20; ++j) {
        float acc = 0.0f;
        for (int u = 0; u < 3; ++u) {
          const int ii = i + (u - 1) * d;
          if (ii < 0 || ii >= 20) continue;
          for (int v = 0; v < 3; ++v) {
            const int jj = j + (v - 1) * d;
            if (jj < 0 || jj >= 20) continue;
            for (int ci = 0; ci < Cin; ++ci)
              acc = fmaf(w[((co * Cin + ci) * 3 + u) * 3 + v], in[ci * 400 + ii * 20 + jj], acc);
          }
        }
        out[co * 400 + i * 20 + j] = bias ? acc + bias[co] : acc;
      }
}

/* AcrE trunk in inference mode (projection.py:706-734 with self.training == False), both ways.
 * feat_out [Q, C*400] (may be NULL) receives relu(bn1(y)); gate_out [Q*C, 1600] (may be NULL; parallel way
 * only) receives the W_gate_e input rows [img ; conv1[c] ; conv2[c] ; conv3[c]]. */
int kgeo_acre_trunk_fwd(const kge_acre_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                        float* feat_out, float* gate_out) {
  const int C = p->in_channels, k = 200, par = p->way == 1;
  const int dil[3] = {p->first_atrous, p->second_atrous, p->third_atrous};
  const float* cw[3] = {p->conv1_weight, p->conv2_weight, p->conv3_weight};
  const float* cb[3] = {p->conv1_bias, p->conv2_bias, p->conv3_bias};
  const int64_t Fw = (int64_t)C * 400;
  if (p->hidden_size != 200 || (p->way != 0 && p->way != 1)) return -2;
  float a0, c0;
  bn_fold(p->bn0_weight[0], p->bn0_bias[0], p->bn0_mean[0], p->bn0_var[0], p->bn0_eps, &a0, &c0);
  float* a1 = (float*)malloc(sizeof(float) * (size_t)C);
  float* c1 = (float*)malloc(sizeof(float) * (size_t)C);
  float* a2 = (float*)malloc(sizeof(float) * (size_t)k);
  float* c2 = (float*)malloc(sizeof(float) * (size_t)k);
  for (int c = 0; c < C; ++c)
    bn_fold(p->bn1_weight[c], p->bn1_bias[c], p->bn1_mean[c], p->bn1_var[c], p->bn1_eps, &a1[c], &c1[c]);
  for (int n = 0; n < k; ++n)
    bn_fold(p->bn2_weight[n], p->bn2_bias[n], p->bn2_mean[n], p->bn2_var[n], p->bn2_eps, &a2[n], &c2[n]);
#pragma omp parallel
  {
    float img[400];
    float* m1 = (float*)malloc(sizeof(float) * (size_t)Fw);
    float* m2 = (float*)malloc(sizeof(float) * (size_t)Fw);
    float* m3 = (float*)malloc(sizeof(float) * (size_t)Fw);
    float* gate = (float*)malloc(sizeof(float) * 1600);
    float* feat = (float*)malloc(sizeof(float) * (size_t)Fw);
#pragma omp for schedule(static)
    for (int64_t q = 0; q < Q; ++q) {
      const float* er = p->ent + e[q] * k;
      const float* rr = p->rel + r[q] * k;
      for (int s = 0; s < 400; ++s) img[s] = fmaf(s < k ? er[s] : rr[s - k], a0, c0);
      if (!par) {
        conv(img, 1, C, dil[0], cw[0], cb[0], m1);
        conv(m1, C, C, dil[1], cw[1], cb[1], m2);
        conv(m2, C, C, dil[2], cw[2], cb[2], m3);
        for (int c = 0; c < C; ++c)
          for (int s = 0; s < 400; ++s)
            feat[c * 400 + s] = fmaxf(fmaf(m3[c * 400 + s] + img[s], a1[c], c1[c]), 0.0f);
      } else {
        conv(img, 1, C, dil[0], cw[0], cb[0], m1);
        conv(img, 1, C, dil[1], cw[1], cb[1], m2);
        conv(img, 1, C, dil[2], cw[2], cb[2], m3);
        for (int c = 0; c < C; ++c) {
          memcpy(gate, img, sizeof(float) * 400);
          memcpy(gate + 400, m1 + c * 400, sizeof(float) * 400);
          memcpy(gate + 800, m2 + c * 400, sizeof(float) * 400);
          memcpy(gate + 1200, m3 + c * 400, sizeof(float) * 400);
          if (gate_out) memcpy(gate_out + (q * C + c) * 1600, gate, sizeof(float) * 1600);
          for (int n = 0; n < 400; ++n) {   /* W_gate_e: one fmaf chain over the 1600 inputs, + bias */
            const float* wr = p->W_gate_e_weight + (int64_t)n * 1600;
            float acc = 0.0f;
            for (int t = 0; t < 1600; ++t) acc = fmaf(gate[t], wr[t], acc);
            acc = acc + p->W_gate_e_bias[n];
            feat[c * 400 + n] = fmaxf(fmaf(acc, a1[c], c1[c]), 0.0f);
          }
        }
      }
      if (feat_out) memcpy(feat_out + q * Fw, feat, sizeof(float) * (size_t)Fw);
      for (int n = 0; n < k; ++n) {   /* Linear: per-slice fmaf chains, slice sums added in order */
        const float* fw = p->fc_weight + (int64_t)n * Fw;
        float total = 0.0f;
        for (int64_t f0 = 0; f0 < Fw; f0 += 512) {
          const int64_t f1 = f0 + 512 < Fw ? f0 + 512 : Fw;
          float acc = 0.0f;
          for (int64_t f = f0; f < f1; ++f) acc = fmaf(feat[f], fw[f], acc);
          total = (f0 == 0) ? acc : total + acc;
        }
        x[q * k + n] = fmaxf(fmaf(total + p->fc_bias[n], a2[n], c2[n]), 0.0f);
      }
    }
    free(m1); free(m2); free(m3); free(gate); free(feat);
  }
  free(a1); free(c1); free(a2); free(c2);
  return 0;
}
