/* tests/oracle_interacte/kge_oracle_interacte.c — TEST INFRASTRUCTURE: scalar C restatement of InteractE's
 * inference trunk in the canonical arithmetic of pykg2vec_b200/csrc/kge_interacte.cuh (the CUDA path must agree
 * with it bit for bit).  Built with gcc -O2 -ffp-contract=off -fno-fast-math -fopenmp -mfma (fmaf() is explicit,
 * nothing else is contracted) by tests/interacte_util.py; the projection tail and its rank counts stay with
 * oracle/.  Nothing in pykg2vec_b200/ can reach it. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* BatchNorm in inference mode folded to fmaf(v, a, c), as ATen folds it (same rule as oracle/kge_oracle.c) */
static void bn_fold(float w, float b, float mean, float var, float eps, float* a, float* c) {
  *a = w / sqrtf(var + eps);
  *c = b - mean * *a;
}

/* InteractE trunk in inference mode: InteractE.forward up to the x.E^T product (projection.py:427-442 with
 * self.training == False).  Canonical arithmetic as pykg2vec_b200/csrc/kge_interacte.cuh states it:
 * img[p][i][j] = fmaf(comb[perm[p][i*W + j]], a0[p], c0[p]) with comb = [ent[e] ; rel[r]];
 * conv output (p, f, i, j) = ks*ks sequential fmaf from 0, row u then column v, of
 * filt[f][u][v] * img[p][(i+u-pad) mod H][(j+v-pad) mod W], then the bn1 fold of channel p*F + f and
 * max(., 0); feature index ((p*F + f)*H + i)*W + j; Linear = one fmaf chain per slice of 512 features, the
 * slice sums added in ascending order, + fc.bias; then the bn2 fold and the ReLU.
 * feat_out [Q, P*F*H*W] (may be NULL) receives the features. */
typedef struct kge_interacte {
  int32_t feature_permutation, num_filters, kernel_size, reshape_height, reshape_width;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  const int64_t* perm;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* conv_filt;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias; const float* bn2_mean; const float* bn2_var;
} kge_interacte_t;

int kgeo_interacte_trunk_fwd(const kge_interacte_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                             float* feat_out) {
  const int P = p->feature_permutation, NF = p->num_filters, ks = p->kernel_size, pad = ks / 2;
  const int H = 2 * p->reshape_width, W = p->reshape_height, k = H * W / 2;
  const int64_t Fw = (int64_t)P * NF * H * W;
  if (ks < 3 || ks % 2 == 0 || pad > H || pad > W) return -2;
  float* a0 = (float*)malloc(sizeof(float) * (size_t)P);
  float* c0 = (float*)malloc(sizeof(float) * (size_t)P);
  float* a1 = (float*)malloc(sizeof(float) * (size_t)P * NF);
  float* c1 = (float*)malloc(sizeof(float) * (size_t)P * NF);
  float* a2 = (float*)malloc(sizeof(float) * (size_t)k);
  float* c2 = (float*)malloc(sizeof(float) * (size_t)k);
  for (int c = 0; c < P; ++c)
    bn_fold(p->bn0_weight[c], p->bn0_bias[c], p->bn0_mean[c], p->bn0_var[c], p->bn0_eps, &a0[c], &c0[c]);
  for (int c = 0; c < P * NF; ++c)
    bn_fold(p->bn1_weight[c], p->bn1_bias[c], p->bn1_mean[c], p->bn1_var[c], p->bn1_eps, &a1[c], &c1[c]);
  for (int n = 0; n < k; ++n)
    bn_fold(p->bn2_weight[n], p->bn2_bias[n], p->bn2_mean[n], p->bn2_var[n], p->bn2_eps, &a2[n], &c2[n]);
#pragma omp parallel
  {
    float* img = (float*)malloc(sizeof(float) * (size_t)P * H * W);
    float* feat = (float*)malloc(sizeof(float) * (size_t)Fw);
#pragma omp for schedule(static)
    for (int64_t q = 0; q < Q; ++q) {
      const float* er = p->ent + e[q] * k;
      const float* rr = p->rel + r[q] * k;
      for (int c = 0; c < P; ++c)
        for (int s = 0; s < H * W; ++s) {
          const int64_t idx = p->perm[(int64_t)c * 2 * k + s];
          img[c * H * W + s] = fmaf(idx < k ? er[idx] : rr[idx - k], a0[c], c0[c]);
        }
      for (int c = 0; c < P; ++c)
        for (int f = 0; f < NF; ++f) {
          const float* w = p->conv_filt + (int64_t)f * ks * ks;
          const int ch = c * NF + f;
          for (int i = 0; i < H; ++i)
            for (int j = 0; j < W; ++j) {
              float acc = 0.0f;
              for (int u = 0; u < ks; ++u) {
                const int si = ((i + u - pad) % H + H) % H;
                for (int v = 0; v < ks; ++v) {
                  const int sj = ((j + v - pad) % W + W) % W;
                  acc = fmaf(w[u * ks + v], img[(c * H + si) * W + sj], acc);
                }
              }
              feat[((int64_t)ch * H + i) * W + j] = fmaxf(fmaf(acc, a1[ch], c1[ch]), 0.0f);
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
    free(img); free(feat);
  }
  free(a0); free(c0); free(a1); free(c1); free(a2); free(c2);
  return 0;
}
