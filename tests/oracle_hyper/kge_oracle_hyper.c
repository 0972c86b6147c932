/* tests/oracle_hyper/kge_oracle_hyper.c — TEST INFRASTRUCTURE: scalar C restatement of HypER's inference
 * trunk in the canonical arithmetic of pykg2vec_b200/csrc/kge_hyper.cuh (the CUDA path must agree with it bit
 * for bit).  Built with gcc -O2 -ffp-contract=off -fno-fast-math -fopenmp -mfma (fmaf() is explicit, nothing
 * else is contracted) by tests/hyper_util.py; the projection tail and its rank counts stay with oracle/.
 * Nothing in pykg2vec_b200/ can reach it. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

/* BatchNorm in inference mode folded to fmaf(v, a, c), as ATen folds it (same rule as oracle/kge_oracle.c) */
static void bn_fold(float w, float b, float mean, float var, float eps, float* a, float* c) {
  *a = w / sqrtf(var + eps);
  *c = b - mean * *a;
}

/* HypER trunk in inference mode: HypER.forward up to the x.E^T product (projection.py:581-606 with
 * self.training == False).  Canonical arithmetic as pykg2vec_b200/csrc/kge_hyper.cuh states it:
 * filters w = fc1(rel[r]) as one fmaf chain over the dr relation features from 0, then + fc1.bias;
 * BatchNorm folded to fmaf(v, a, c); conv output (c, j) = 9 sequential fmaf from 0 of w[9c+t] * v[j+t]
 * in t order, then the bn1 fold (no conv bias, no ReLU), feature index c*(de-8) + j; Linear = one fmaf
 * chain per slice of 512 features, the slice sums added in ascending order, + fc.bias; then the bn2
 * fold and the ReLU.  filt_out [num_rel, 288] and feat_out [Q, 32*(de-8)] (each may be NULL) receive
 * the intermediate filter table and features. */
typedef struct kge_hyper {
  int32_t ent_hidden_size, rel_hidden_size;
  int64_t num_rel;
  float bn0_eps, bn1_eps, bn2_eps;
  const float* ent; const float* rel;
  const float* bn0_weight; const float* bn0_bias; const float* bn0_mean; const float* bn0_var;
  const float* fc1_weight; const float* fc1_bias;
  const float* bn1_weight; const float* bn1_bias; const float* bn1_mean; const float* bn1_var;
  const float* fc_weight; const float* fc_bias;
  const float* bn2_weight; const float* bn2_bias; const float* bn2_mean; const float* bn2_var;
} kge_hyper_t;

static void hyper_filters(const kge_hyper_t* p, int64_t rr, float* w) {
  const int dr = p->rel_hidden_size;
  const float* rv = p->rel + rr * dr;
  for (int o = 0; o < 288; ++o) {
    const float* fw = p->fc1_weight + (int64_t)o * dr;
    float acc = 0.0f;
    for (int i = 0; i < dr; ++i) acc = fmaf(rv[i], fw[i], acc);
    w[o] = acc + p->fc1_bias[o];
  }
}

int kgeo_hyper_trunk_fwd(const kge_hyper_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                         float* filt_out, float* feat_out) {
  const int de = p->ent_hidden_size, Wo = de - 8;
  const int64_t F = (int64_t)32 * Wo;
  float a0, c0, a1[32], c1[32];
  bn_fold(p->bn0_weight[0], p->bn0_bias[0], p->bn0_mean[0], p->bn0_var[0], p->bn0_eps, &a0, &c0);
  for (int c = 0; c < 32; ++c)
    bn_fold(p->bn1_weight[c], p->bn1_bias[c], p->bn1_mean[c], p->bn1_var[c], p->bn1_eps, &a1[c], &c1[c]);
  float* a2 = (float*)malloc(sizeof(float) * (size_t)de);
  float* c2 = (float*)malloc(sizeof(float) * (size_t)de);
  for (int n = 0; n < de; ++n)
    bn_fold(p->bn2_weight[n], p->bn2_bias[n], p->bn2_mean[n], p->bn2_var[n], p->bn2_eps, &a2[n], &c2[n]);
  if (filt_out)
    for (int64_t rr = 0; rr < p->num_rel; ++rr) hyper_filters(p, rr, filt_out + rr * 288);
#pragma omp parallel
  {
    float* v = (float*)malloc(sizeof(float) * (size_t)de);
    float* feat = (float*)malloc(sizeof(float) * (size_t)F);
    float w[288];
#pragma omp for schedule(static)
    for (int64_t q = 0; q < Q; ++q) {
      const float* er = p->ent + e[q] * de;
      for (int i = 0; i < de; ++i) v[i] = fmaf(er[i], a0, c0);
      hyper_filters(p, r[q], w);
      for (int c = 0; c < 32; ++c)
        for (int j = 0; j < Wo; ++j) {
          float acc = 0.0f;
          for (int t = 0; t < 9; ++t) acc = fmaf(w[c * 9 + t], v[j + t], acc);
          feat[c * Wo + j] = fmaf(acc, a1[c], c1[c]);
        }
      if (feat_out) memcpy(feat_out + q * F, feat, sizeof(float) * (size_t)F);
      for (int n = 0; n < de; ++n) {   /* Linear: per-slice fmaf chains, slice sums added in order */
        const float* fw = p->fc_weight + (int64_t)n * F;
        float total = 0.0f;
        for (int64_t f0 = 0; f0 < F; f0 += 512) {
          const int64_t f1 = f0 + 512 < F ? f0 + 512 : F;
          float acc = 0.0f;
          for (int64_t f = f0; f < f1; ++f) acc = fmaf(feat[f], fw[f], acc);
          total = (f0 == 0) ? acc : total + acc;
        }
        x[q * de + n] = fmaxf(fmaf(total + p->fc_bias[n], a2[n], c2[n]), 0.0f);
      }
    }
    free(v); free(feat);
  }
  free(a2); free(c2);
  return 0;
}
