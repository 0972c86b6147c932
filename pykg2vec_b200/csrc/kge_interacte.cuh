// kge_interacte.cuh — InteractE's trunk in inference mode (InteractE.forward, pykg2vec/models/projection.py:425-442
// with self.training == False: dropouts are identities, bn0 / bn1 / bn2 use their running statistics):
//     comb = [ent[e] ; rel[r]]                        2k values, k = reshape_width * reshape_height
//     img[p][i][j] = bn0_p(comb[perm[p][i*W + j]])    P chequer-permuted images of H = 2*reshape_width rows and
//                                                     W = reshape_height columns
//     circular conv ks x ks (pad = ks/2 on both axes, filter f on image p -> channel p*F + f, no conv bias)
//     -> bn1 -> relu -> flatten channel-major          (interacte_feature_kernel below)
//     x = relu(bn2(feat . fc.weight^T + fc.bias))     (ConvE's sliced Linear GEMM + hyper_fc_combine_kernel)
// Canonical arithmetic (restated by tests/oracle_interacte/kge_oracle_interacte.c, bit for bit):
//     BatchNorm(v) = fma(v, a, c) with a = w / sqrt(var + eps), c = b - mean * a (bn_fold);
//     conv output (p, f, i, j) = ks*ks sequential fma from 0 in tap order (row u, then column v) of
//     filt[f][u][v] * img[p][(i + u - pad) mod H][(j + v - pad) mod W], then the bn1 fold, then max(., 0);
//     feature index ((p*F + f)*H + i)*W + j;
//     Linear and combine = HypER's (kge_hyper.cuh): one fma chain per slice of CONVE_FC_SLICE features, slice
//     sums added in ascending order, then + fc.bias, then the bn2 fold, then relu.
#pragma once
#include "kge_hyper.cuh"

namespace kge {

constexpr int INTERACTE_THREADS = 256;
constexpr int INTERACTE_FB = 8;                    // filters per thread (the filter bank is padded to a multiple)
constexpr int INTERACTE_SMEM_MAX = 227 * 1024;     // bytes: the per-block opt-in maximum of sm_90

struct InteracteFeat {
  const float* ent; const float* rel;   // [N, k], [R, k]
  const int64_t* perm;                  // [P, 2k]
  const int64_t* e; const int64_t* r;
  int P, F, ks, H, W;                   // H = 2 * reshape_width, W = reshape_height
  const float* bn0_w; const float* bn0_b; const float* bn0_mean; const float* bn0_var; float bn0_eps;
  const float* conv_filt;               // [F, 1, ks, ks]
  const float* bn1_w; const float* bn1_b; const float* bn1_mean; const float* bn1_var; float bn1_eps;
  float* feat;                          // [Q, P*F*H*W]
};

__host__ __device__ inline int interacte_fpad(int F) { return (F + INTERACTE_FB - 1) / INTERACTE_FB * INTERACTE_FB; }
inline long long interacte_feat_width(int P, int F, int H, int W) { return (long long)P * F * H * W; }

// Shared memory, in floats: the filter bank transposed to [ks*ks][Fpad] (zero columns f >= F), the bn1 folds
// a1 / c1 [P][Fpad] each, then the P circularly padded images [(H + 2 pad)][(W + 2 pad)].
struct InteracteSmem { long long wt, a1, c1, img, total; };

__host__ __device__ inline InteracteSmem interacte_smem(int P, int F, int ks, int H, int W) {
  const long long Fp = interacte_fpad(F), pad = ks / 2;
  InteracteSmem S;
  S.wt = 0;
  S.a1 = (long long)ks * ks * Fp;
  S.c1 = S.a1 + P * Fp;
  S.img = S.c1 + P * Fp;
  S.total = S.img + P * (H + 2 * pad) * (W + 2 * pad);
  return S;
}

// one CTA per query.  A thread computes INTERACTE_FB consecutive filters at one pixel: per tap one image value
// (consecutive pixels across the warp) and two float4 filter reads (the same address across the warp).
__global__ void __launch_bounds__(INTERACTE_THREADS) interacte_feature_kernel(const InteracteFeat p) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else   // host emulation (tests/emu): __shared__ is a function-local static there, so it needs a fixed size
  __shared__ float4 smem_f4[INTERACTE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const int q = blockIdx.x, tid = threadIdx.x;
  const int P = p.P, F = p.F, ks = p.ks, H = p.H, W = p.W, pad = ks / 2;
  const int Fp = interacte_fpad(F), k = H * W / 2, taps = ks * ks;
  const int Hp = H + 2 * pad, Wp = W + 2 * pad, plane = Hp * Wp;
  const InteracteSmem S = interacte_smem(P, F, ks, H, W);
  float* wt = sm + S.wt;
  float* a1 = sm + S.a1;
  float* c1 = sm + S.c1;
  float* img = sm + S.img;
  for (int i = tid; i < taps * Fp; i += INTERACTE_THREADS) {
    const int t = i / Fp, f = i - t * Fp;
    wt[i] = f < F ? __ldg(p.conv_filt + (long long)f * taps + t) : 0.f;
  }
  for (int i = tid; i < P * Fp; i += INTERACTE_THREADS) {
    const int pp = i / Fp, f = i - pp * Fp, c = pp * F + f;
    if (f < F)
      bn_fold(__ldg(p.bn1_w + c), __ldg(p.bn1_b + c), __ldg(p.bn1_mean + c), __ldg(p.bn1_var + c), p.bn1_eps, a1[i],
              c1[i]);
    else
      a1[i] = c1[i] = 0.f;
  }
  const float* er = p.ent + __ldg(p.e + q) * (long long)k;
  const float* rr = p.rel + __ldg(p.r + q) * (long long)k;
  for (int i = tid; i < P * plane; i += INTERACTE_THREADS) {
    const int pp = i / plane, rem = i - pp * plane, pi = rem / Wp, pj = rem - pi * Wp;
    int si = pi - pad, sj = pj - pad;      // circular padding: pad <= H and pad <= W, so one wrap suffices
    si += si < 0 ? H : (si >= H ? -H : 0);
    sj += sj < 0 ? W : (sj >= W ? -W : 0);
    const int64_t idx = __ldg(p.perm + (long long)pp * 2 * k + si * W + sj);
    const float v = idx < k ? __ldg(er + idx) : __ldg(rr + (idx - k));
    float a0, c0;
    bn_fold(__ldg(p.bn0_w + pp), __ldg(p.bn0_b + pp), __ldg(p.bn0_mean + pp), __ldg(p.bn0_var + pp), p.bn0_eps, a0,
            c0);
    img[i] = ffma(v, a0, c0);
  }
  __syncthreads();
  const int HW = H * W, G = Fp / INTERACTE_FB, items = P * G * HW;
  float* out = p.feat + (long long)q * P * F * HW;
  for (int it = tid; it < items; it += INTERACTE_THREADS) {
    const int pg = it / HW, pix = it - pg * HW, pp = pg / G, g = pg - pp * G;
    const int i = pix / W, j = pix - i * W;
    const float* ip = img + pp * plane + i * Wp + j;
    const float* wp = wt + g * INTERACTE_FB;
    float acc[INTERACTE_FB];
#pragma unroll
    for (int b = 0; b < INTERACTE_FB; ++b) acc[b] = 0.f;
    for (int u = 0; u < ks; ++u) {
      const float* row = ip + u * Wp;
      const float* wrow = wp + u * ks * Fp;
      for (int v = 0; v < ks; ++v) {
        const float x = row[v];
        const float4 w0 = *reinterpret_cast<const float4*>(wrow + v * Fp);
        const float4 w1 = *reinterpret_cast<const float4*>(wrow + v * Fp + 4);
        acc[0] = ffma(w0.x, x, acc[0]); acc[1] = ffma(w0.y, x, acc[1]);
        acc[2] = ffma(w0.z, x, acc[2]); acc[3] = ffma(w0.w, x, acc[3]);
        acc[4] = ffma(w1.x, x, acc[4]); acc[5] = ffma(w1.y, x, acc[5]);
        acc[6] = ffma(w1.z, x, acc[6]); acc[7] = ffma(w1.w, x, acc[7]);
      }
    }
    const int f0 = g * INTERACTE_FB;
#pragma unroll
    for (int b = 0; b < INTERACTE_FB; ++b) {
      const int f = f0 + b;
      if (f < F)
        out[((long long)(pp * F + f) * H + i) * W + j] = fmaxf(ffma(acc[b], a1[pp * Fp + f], c1[pp * Fp + f]), 0.f);
    }
  }
}

// ---- launch plan: plain C++ shared by the C-ABI launcher (kge_proj.cu) and the CPU emulation test ---------
// Workspace, in floats: the features [Q, P*F*H*W], then the Linear layer's slice partials [slices, Q, k].
// The GEMM reads the features with float4 loads only where proj_vec_ok allows; the partials are written and
// read one float at a time.
struct InteracteLayout { long long feat, partial, total; };

inline InteracteLayout interacte_layout(long long Q, int P, int F, int H, int W) {
  const long long Fw = interacte_feat_width(P, F, H, W);
  InteracteLayout L;
  L.feat = 0;
  L.partial = Q * Fw;
  L.total = L.partial + (long long)conve_fc_slices(Fw) * Q * (H * W / 2);
  return L;
}

}  // namespace kge
