// kge_hyper.cuh — HypER's trunk in inference mode (HypER.forward, pykg2vec/models/projection.py:581-606
// with self.training == False: dropouts are identities, bn0 / bn1 / bn2 use their running statistics):
//     filt[R, 288] = rel . fc1.weight^T + fc1.bias     every relation's 32 filters of width 9 (the
//                                                     hypernetwork), one launch of the tiled GEMM of
//                                                     kge_proj.cuh
//     bn0 -> per-query conv 1x9 (1 -> 32 channels, the query's own filters) -> bn1 -> flatten
//                                                    (hyper_feature_kernel below; NO ReLU after bn1)
//     x = relu(bn2(feat . fc.weight^T + fc.bias))     (ConvE's sliced Linear GEMM + the combine kernel
//                                                     below; bn2 IS applied in eval mode, unlike ConvE)
// Canonical arithmetic (restated by tests/oracle_hyper/kge_oracle_hyper.c, bit for bit):
//     filter = one sequential fma chain over the dr relation features from 0, then + fc1.bias;
//     BatchNorm(v) = fma(v, a, c) with a = w / sqrt(var + eps), c = b - mean * a (bn_fold);
//     conv output (c, j) = 9 sequential fma from 0 in tap order t = 0..8 of w[9c + t] * v[j + t],
//     then the bn1 fold (no conv bias); feature index c * (de - 8) + j (channel-major, the
//     view / permute chain of projection.py:588-598);
//     Linear = ConvE's: one fma chain per slice of CONVE_FC_SLICE features, slice sums added in
//     ascending order, then + fc.bias; then the bn2 fold, then relu.
#pragma once
#include "kge_conve.cuh"

namespace kge {

constexpr int HYPER_CH = 32;          // out_channels (projection.py:529)
constexpr int HYPER_FW = 9;           // filt_w; filt_h = 1
constexpr int HYPER_FILT = HYPER_CH * HYPER_FW;   // fc1 output width, 288
constexpr int HYPER_THREADS = 256;
constexpr int HYPER_MAX_DE = 4096;    // entity row held in shared memory

struct HyperFeat {
  const float* ent; const float* filt;   // [N, de], [R, 288]
  const int64_t* e; const int64_t* r;
  int de;
  const float* bn0_w; const float* bn0_b; const float* bn0_mean; const float* bn0_var; float bn0_eps;
  const float* bn1_w; const float* bn1_b; const float* bn1_mean; const float* bn1_var; float bn1_eps;
  float* feat;                           // [Q, 32 * (de - 8)]
};

inline long long hyper_feat_width(int de) { return (long long)HYPER_CH * (de - HYPER_FW + 1); }

// one CTA per query
__global__ void __launch_bounds__(HYPER_THREADS) hyper_feature_kernel(const HyperFeat p) {
  __shared__ float v[HYPER_MAX_DE];
  __shared__ float w[HYPER_FILT];
  __shared__ float a1[HYPER_CH], c1[HYPER_CH];
  const int q = blockIdx.x, tid = threadIdx.x;
  const int de = p.de, Wo = de - HYPER_FW + 1, n = HYPER_CH * Wo;
  float a0, c0;
  bn_fold(__ldg(p.bn0_w), __ldg(p.bn0_b), __ldg(p.bn0_mean), __ldg(p.bn0_var), p.bn0_eps, a0, c0);
  const float* er = p.ent + __ldg(p.e + q) * (long long)de;
  const float* fr = p.filt + __ldg(p.r + q) * (long long)HYPER_FILT;
  for (int i = tid; i < de; i += HYPER_THREADS) v[i] = ffma(__ldg(er + i), a0, c0);
  for (int i = tid; i < HYPER_FILT; i += HYPER_THREADS) w[i] = __ldg(fr + i);
  if (tid < HYPER_CH)
    bn_fold(__ldg(p.bn1_w + tid), __ldg(p.bn1_b + tid), __ldg(p.bn1_mean + tid), __ldg(p.bn1_var + tid),
            p.bn1_eps, a1[tid], c1[tid]);
  __syncthreads();
  float* out = p.feat + (long long)q * n;
  for (int o = tid; o < n; o += HYPER_THREADS) {
    const int c = o / Wo, j = o - c * Wo;
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < HYPER_FW; ++t) acc = ffma(w[c * HYPER_FW + t], v[j + t], acc);
    out[o] = ffma(acc, a1[c], c1[c]);
  }
}

// x[i] = relu(bn2(((P_0[i] + P_1[i]) + ... + P_{S-1}[i]) + fc_b[i % k]))
__global__ void __launch_bounds__(256)
hyper_fc_combine_kernel(const float* __restrict__ partial, int slices, long long n, int k,
                        const float* __restrict__ fc_b, const float* __restrict__ bn2_w,
                        const float* __restrict__ bn2_b, const float* __restrict__ bn2_mean,
                        const float* __restrict__ bn2_var, float bn2_eps, float* __restrict__ x) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const int col = (int)(i % k);
  float acc = __ldg(partial + i);
  for (int s = 1; s < slices; ++s) acc = fadd(acc, __ldg(partial + (long long)s * n + i));
  float a2, c2;
  bn_fold(__ldg(bn2_w + col), __ldg(bn2_b + col), __ldg(bn2_mean + col), __ldg(bn2_var + col), bn2_eps, a2, c2);
  x[i] = fmaxf(ffma(fadd(acc, __ldg(fc_b + col)), a2, c2), 0.f);
}

// ---- launch plans: plain C++ shared by the C-ABI launcher (kge_proj.cu) and the CPU emulation test ---
// Workspace, in floats: the filter table [R, 288], the features [Q, F], the Linear layer's slice
// partials [slices, Q, de].  Every region starts 16-byte aligned (288 and F are multiples of 4).
struct HyperLayout { long long filt, feat, partial, total; };

inline HyperLayout hyper_layout(long long R, long long Q, int de) {
  const long long F = hyper_feat_width(de);
  HyperLayout L;
  L.filt = 0;
  L.feat = R * HYPER_FILT;
  L.partial = L.feat + Q * F;
  L.total = L.partial + (long long)conve_fc_slices(F) * Q * de;
  return L;
}

// filt[R, 288] = rel[R, dr] . fc1_w[288, dr]^T + fc1_b   (no activation)
inline ProjLaunch hyper_plan_filters(const float* rel, const float* fc1_w, const float* fc1_b, long long R, int dr,
                                     float* filt) {
  ProjLaunch L = proj_plan_fwd(rel, fc1_w, fc1_b, R, HYPER_FILT, dr, filt, PROJ_TILE_64x64);
  L.g.act = ACT_NONE;
  return L;
}

}  // namespace kge
