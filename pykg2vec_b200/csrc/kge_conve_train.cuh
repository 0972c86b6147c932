// kge_conve_train.cuh — ConvE's trunk in TRAINING mode (pykg2vec/models/projection.py:86-99 with
// self.training == True), forward and backward, launched from kge_proj.cu (kge_conve_train_*).
// Per query q of a group of B queries (one direction of train_step_projection):
//     img[2*h2, h1] = [ent[e] ; rel[r]]
//     bn0 (batch statistics over the group's B * 2k values) -> * noise0[q, :] (inp_drop)
//     conv 3x3 (1 -> 32, no padding) + bias -> z1 -> bn1 (per channel, over B * Ho * Wo) -> relu
//     * noise1[q, c] (feat_drop = Dropout2d: one value per (query, channel)) -> feat [F]
//     hpre = (feat . fc.weight^T + fc.bias) * noise2[q, :] (hidden_drop)
//     x = relu(bn2(hpre))   (per feature, over the group's B rows)
// Kernels (one CTA per query unless noted):
//   conve_tr_gather_kernel      img (raw) + per-query (sum, centred sum of squares) of its 2k values
//   conve_tr_bn_stats_kernel    thread per channel: the group's mean / invstd from the per-query partials, running
//                               statistics updated group after group (= one BatchNorm call per group, in order)
//   conve_tr_conv_kernel        bn0 + noise0 + conv -> z1, per-query per-channel partials of z1
//   conve_tr_feat_kernel        feat = relu(bn1(z1)) * noise1 (elementwise)
//   (tiled GEMM, kge_proj.cuh)  the Linear layer in CONVE_FC_SLICE slices (conve_plan_fc)
//   conve_tr_fc_combine_kernel  hpre = (slices in ascending order + fc.bias) * noise2
//   conve_tr_bn2_kernel         thread per feature: bn2's statistics (two-pass), running statistics, x
// backward (gradients ACCUMULATED into dense buffers shaped like the parameters):
//   conve_tr_bn2_bwd_kernel     thread per feature: relu mask, bn2 backward, * noise2 -> dh; d bn2.*, d fc.bias
//   (tiled GEMM)                d fc.weight += dh^T . feat (one slice, atomic epilogue), dfeat = dh . fc.weight
//   conve_tr_bn1_bwd_part_kernel  * noise1, relu mask -> g1 (in place), per-query per-channel (sum g1, sum g1 xhat)
//   conve_tr_reduce_kernel      thread per channel: the partials summed over each group's queries in ascending
//                               order -> d bn.weight, d bn.bias (bn1, then bn0)
//   conve_tr_conv_bwd_kernel    bn1 backward -> dz1 (in place); per-query d conv.weight / d conv.bias partials;
//                               transposed conv -> d img, * noise0; per-query bn0 partials
//   conve_tr_colsum_kernel      d conv.weight / d conv.bias: partials summed over queries in ascending order
//   conve_tr_bn0_bwd_kernel     bn0 backward -> grad_ent[e] / grad_rel[r] (float atomics: ids repeat)
//
// Canonical arithmetic of the forward (DESIGN.md §3, ConvE training), restated by tests/oracle_conve_train bit for
// bit; nothing in it depends on the grid or on the other groups of the call, so x and the running statistics are
// bit-reproducible and a call over G groups equals G calls:
//   CTA sum       one value per thread (thread t accumulates elements t, t+256, ... in increasing order), xor
//                 butterfly 16, 8, 4, 2, 1 inside each warp, then the 8 warp sums added in ascending warp order
//   warp sum      lane l accumulates elements l, l+32, ... in increasing order, xor butterfly 16 .. 1
//   per query     s = sum v (CTA sum for bn0, warp sum per channel for bn1), m = s / n_q, m2 = sum (v - m)^2
//   group stats   S = sum_q s_q, q ascending; mean = S / n; M2 = sum_q (m2_q + n_q (m_q - mean)^2), q ascending;
//                 var = M2 / n; invstd = 1 / sqrt(var + eps).  bn2: n_q = 1 (two passes over the B values)
//   normalise     y = fma((v - mean) * invstd, weight, bias)
//   running       rm = (1 - mom) * rm + mom * mean; rv = (1 - mom) * rv + mom * (var * n / (n - 1)), group 0 first
//   conv          9 sequential fma from 0 in (di, dj) row-major order, then + conv bias (as kge_conve.cuh)
//   Linear        kge_conve.cuh's sliced chain: slice sums added in ascending slice order, then + fc.bias
// The backward's sums over queries are ordered too except for the entity / relation scatter (float atomics), and
// d fc.weight's single GEMM slice adds each element once into the (caller-zeroed) buffer.
#pragma once
#include "kge_conve.cuh"

namespace kge {

constexpr int CONVE_TR_THREADS = 256;
constexpr int CONVE_TAPS = CONVE_CH * 9;   // conv2d_1.weight elements

struct ConveTrain {
  const float* ent; const float* rel;
  const int64_t* e; const int64_t* r;
  int k, h2, h1;                 // image 2*h2 x h1 (k == h2 * h1)
  long long Q, B;                // rows, rows per group
  const float* bn0_w; const float* bn0_b;
  const float* conv_w; const float* conv_b;
  const float* bn1_w; const float* bn1_b;
  const float* bn2_w; const float* bn2_b;
  const float* noise0;           // [Q, 2k] or NULL
  const float* noise1;           // [Q, 32] or NULL
  const float* noise2;           // [Q, k] or NULL
  // workspace (forward writes, backward reads; the backward's scratch follows)
  float* img;                    // [Q, 2k]
  float* z1;                     // [Q, F]
  float* feat;                   // [Q, F]
  float* hpre;                   // [Q, k]
  float* st0;                    // [G, 2]      bn0 (mean, invstd) of each group
  float* st1;                    // [G, 32, 2]
  float* st2;                    // [G, k, 2]
  float* part0;                  // [Q, 2]      per-query partials of bn0 (forward, then backward)
  float* part1;                  // [Q, 32, 2]  of bn1
  float* red0;                   // [G, 1, 2]   backward: group sums (sum g, sum g xhat) of bn0
  float* red1;                   // [G, 32, 2]  of bn1
  float* dz;                     // [Q, F]      d feat -> g1 -> dz1
  float* dimg;                   // [Q, 2k]     d (bn0 output)
  float* pw;                     // [Q, 288]    per-query d conv.weight
  float* pb;                     // [Q, 32]     per-query d conv.bias
};

struct ConveTrainLayout {
  long long img, z1, feat, partial, hpre, st0, st1, st2, part0, part1, red0, red1, dh, dz, dimg, pw, pb, total;
};

// float offsets of the workspace regions, each 64-float aligned (16-byte loads of the GEMM operands)
inline ConveTrainLayout conve_train_layout(long long Q, long long B, int k, int h1) {
  const int h2 = k / h1;
  const long long F = conve_feat_width(h2, h1), S = conve_fc_slices(F), G = Q / B, n0 = 2ll * k;
  ConveTrainLayout L{};
  long long o = 0;
  auto take = [&o](long long n) { const long long at = o; o += (n + 63) / 64 * 64; return at; };
  L.img = take(Q * n0); L.z1 = take(Q * F); L.feat = take(Q * F); L.partial = take(S * Q * k); L.hpre = take(Q * k);
  L.st0 = take(G * 2); L.st1 = take(G * CONVE_CH * 2); L.st2 = take(G * k * 2);
  L.part0 = take(Q * 2); L.part1 = take(Q * CONVE_CH * 2);
  L.red0 = take(G * 2); L.red1 = take(G * CONVE_CH * 2);
  L.dh = take(Q * k); L.dz = take(Q * F); L.dimg = take(Q * n0); L.pw = take(Q * CONVE_TAPS); L.pb = take(Q * CONVE_CH);
  L.total = o;
  return L;
}

KGE_DEV float conve_warp_sum(float v) {
#pragma unroll
  for (int off = 16; off; off >>= 1) v = fadd(v, __shfl_xor_sync(0xffffffffu, v, off));
  return v;
}

// the CTA sum of one value per thread (every thread gets it); sh: CONVE_TR_THREADS / 32 floats, barriers inside
KGE_DEV float conve_block_sum(float v, float* sh) {
  v = conve_warp_sum(v);
  __syncthreads();   // sh is free: every thread is past its last read of an earlier call
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
  __syncthreads();
  float s = sh[0];
#pragma unroll
  for (int w = 1; w < CONVE_TR_THREADS / 32; ++w) s = fadd(s, sh[w]);
  return s;
}

KGE_DEV float conve_bn_apply(float v, float mean, float invstd, float w, float b) {
  return ffma(fmul(fsub(v, mean), invstd), w, b);
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) conve_tr_gather_kernel(const ConveTrain a) {
  __shared__ float sh[CONVE_TR_THREADS / 32];
  const long long q = blockIdx.x;
  const int k = a.k, n0 = 2 * k, tid = threadIdx.x;
  const float* er = a.ent + __ldg(a.e + q) * (long long)k;
  const float* rr = a.rel + __ldg(a.r + q) * (long long)k;
  float* out = a.img + q * n0;
  float s = 0.f;
  for (int i = tid; i < n0; i += CONVE_TR_THREADS) {
    const float v = i < k ? __ldg(er + i) : __ldg(rr + (i - k));
    out[i] = v;
    s = fadd(s, v);
  }
  s = conve_block_sum(s, sh);
  const float m = __fdiv_rn(s, (float)n0);
  float m2 = 0.f;
  for (int i = tid; i < n0; i += CONVE_TR_THREADS) {   // this thread's own elements: no barrier needed
    const float d = fsub(out[i], m);
    m2 = ffma(d, d, m2);
  }
  m2 = conve_block_sum(m2, sh);
  if (tid == 0) { a.part0[q * 2] = s; a.part0[q * 2 + 1] = m2; }
}

// thread c < C: for each group g in ascending order, the statistics of channel c from the per-query partials
// part[q][c] = (sum, centred sum of squares) of nq values each; st[g][c] = (mean, invstd); running stats updated
__global__ void __launch_bounds__(256)
conve_tr_bn_stats_kernel(const float* __restrict__ part, long long Q, long long B, int C, float nq, float eps,
                         float mom, float* __restrict__ st, float* rmean, float* rvar) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  const long long G = Q / B;
  const float n = fmul((float)B, nq);
  for (long long g = 0; g < G; ++g) {
    const float* p = part + (g * B * C + c) * 2;
    float S = 0.f;
    for (long long i = 0; i < B; ++i) S = fadd(S, p[i * C * 2]);
    const float mean = __fdiv_rn(S, n);
    float M2 = 0.f;
    for (long long i = 0; i < B; ++i) {
      const float d = fsub(__fdiv_rn(p[i * C * 2], nq), mean);
      M2 = fadd(M2, ffma(fmul(nq, d), d, p[i * C * 2 + 1]));
    }
    const float var = __fdiv_rn(M2, n);
    st[(g * C + c) * 2] = mean;
    st[(g * C + c) * 2 + 1] = __fdiv_rn(1.0f, __fsqrt_rn(fadd(var, eps)));
    if (rmean) {
      rmean[c] = ffma(mom, mean, fmul(fsub(1.0f, mom), rmean[c]));
      rvar[c] = ffma(mom, __fdiv_rn(fmul(var, n), fsub(n, 1.0f)), fmul(fsub(1.0f, mom), rvar[c]));
    }
  }
}

// bn0 + noise0 into shared memory (the conv input), shared by the forward conv and its backward
KGE_DEV void conve_tr_conv_input(const ConveTrain& a, long long q, float* xin) {
  const int n0 = 2 * a.k;
  const long long g = q / a.B;
  const float mean = a.st0[g * 2], invstd = a.st0[g * 2 + 1], w = __ldg(a.bn0_w), b = __ldg(a.bn0_b);
  for (int i = threadIdx.x; i < n0; i += CONVE_TR_THREADS) {
    float v = conve_bn_apply(a.img[q * n0 + i], mean, invstd, w, b);
    if (a.noise0) v = fmul(v, __ldg(a.noise0 + q * n0 + i));
    xin[i] = v;
  }
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) conve_tr_conv_kernel(const ConveTrain a) {
  __shared__ float xin[CONVE_MAX_IMAGE];
  __shared__ float wgt[CONVE_TAPS];
  __shared__ float cb[CONVE_CH];
  const long long q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int W = a.h1, Ho = 2 * a.h2 - 2, Wo = a.h1 - 2, plane = Ho * Wo, F = CONVE_CH * plane;
  conve_tr_conv_input(a, q, xin);
  for (int i = tid; i < CONVE_TAPS; i += CONVE_TR_THREADS) wgt[i] = __ldg(a.conv_w + i);
  if (tid < CONVE_CH) cb[tid] = __ldg(a.conv_b + tid);
  __syncthreads();
  float* out = a.z1 + q * F;
  for (int o = tid; o < F; o += CONVE_TR_THREADS) {
    const int c = o / plane, rem = o - c * plane;
    const int i = rem / Wo, j = rem - i * Wo;
    float acc = 0.f;
#pragma unroll
    for (int di = 0; di < 3; ++di)
#pragma unroll
      for (int dj = 0; dj < 3; ++dj) acc = ffma(wgt[c * 9 + di * 3 + dj], xin[(i + di) * W + j + dj], acc);
    out[o] = fadd(acc, cb[c]);
  }
  __syncthreads();   // z1 of this query is complete (global writes of the CTA are visible after the barrier)
  for (int c = warp; c < CONVE_CH; c += CONVE_TR_THREADS / 32) {
    const float* zc = out + c * plane;
    float s = 0.f;
    for (int p = lane; p < plane; p += 32) s = fadd(s, zc[p]);
    s = conve_warp_sum(s);
    const float m = __fdiv_rn(s, (float)plane);
    float m2 = 0.f;
    for (int p = lane; p < plane; p += 32) {
      const float d = fsub(zc[p], m);
      m2 = ffma(d, d, m2);
    }
    m2 = conve_warp_sum(m2);
    if (lane == 0) { a.part1[(q * CONVE_CH + c) * 2] = s; a.part1[(q * CONVE_CH + c) * 2 + 1] = m2; }
  }
}

KGE_DEV float conve_tr_bn1(const ConveTrain& a, long long q, int c, float z) {
  const float* st = a.st1 + ((q / a.B) * CONVE_CH + c) * 2;
  return conve_bn_apply(z, st[0], st[1], __ldg(a.bn1_w + c), __ldg(a.bn1_b + c));
}

__global__ void __launch_bounds__(256) conve_tr_feat_kernel(const ConveTrain a, long long F, int plane) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.Q * F) return;
  const long long q = i / F;
  const int c = (int)((i - q * F) / plane);
  float v = fmaxf(conve_tr_bn1(a, q, c, __ldg(a.z1 + i)), 0.f);
  if (a.noise1) v = fmul(v, __ldg(a.noise1 + q * CONVE_CH + c));
  a.feat[i] = v;
}

// hpre[i] = (((P_0[i] + P_1[i]) + ... + P_{S-1}[i]) + fc_b[i % k]) * noise2[i]
__global__ void __launch_bounds__(256)
conve_tr_fc_combine_kernel(const float* __restrict__ partial, int slices, long long n, int k,
                           const float* __restrict__ fc_b, const float* __restrict__ noise2, float* __restrict__ hpre) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  float acc = __ldg(partial + i);
  for (int s = 1; s < slices; ++s) acc = fadd(acc, __ldg(partial + (long long)s * n + i));
  acc = fadd(acc, __ldg(fc_b + (int)(i % k)));
  hpre[i] = noise2 ? fmul(acc, __ldg(noise2 + i)) : acc;
}

// thread j < k: bn2 over each group's B rows (two passes), running statistics, x = relu(bn2(hpre))
__global__ void __launch_bounds__(256)
conve_tr_bn2_kernel(const ConveTrain a, float eps, float mom, float* rmean, float* rvar, float* __restrict__ x) {
  const int j = blockIdx.x * 256 + threadIdx.x, k = a.k;
  if (j >= k) return;
  const long long G = a.Q / a.B;
  const float n = (float)a.B, w = __ldg(a.bn2_w + j), b = __ldg(a.bn2_b + j);
  for (long long g = 0; g < G; ++g) {
    const float* h = a.hpre + g * a.B * k + j;
    float S = 0.f;
    for (long long i = 0; i < a.B; ++i) S = fadd(S, h[i * k]);
    const float mean = __fdiv_rn(S, n);
    float M2 = 0.f;
    for (long long i = 0; i < a.B; ++i) {
      const float d = fsub(h[i * k], mean);
      M2 = ffma(d, d, M2);
    }
    const float var = __fdiv_rn(M2, n), invstd = __fdiv_rn(1.0f, __fsqrt_rn(fadd(var, eps)));
    a.st2[(g * k + j) * 2] = mean;
    a.st2[(g * k + j) * 2 + 1] = invstd;
    if (rmean) {
      rmean[j] = ffma(mom, mean, fmul(fsub(1.0f, mom), rmean[j]));
      rvar[j] = ffma(mom, __fdiv_rn(fmul(var, n), fsub(n, 1.0f)), fmul(fsub(1.0f, mom), rvar[j]));
    }
    float* xo = x + g * a.B * k + j;
    for (long long i = 0; i < a.B; ++i) xo[i * k] = fmaxf(conve_bn_apply(h[i * k], mean, invstd, w, b), 0.f);
  }
}

// ---- backward ------------------------------------------------------------------------------------------------

// BatchNorm's input gradient from the output gradient gy and xhat, given the group sums sg = sum gy and
// sgx = sum gy xhat over n values:  w * invstd * (gy - sg / n - xhat * sgx / n)
KGE_DEV float conve_bn_bwd(float gy, float xhat, float sg, float sgx, float inv_n, float w, float invstd) {
  return fmul(fmul(w, invstd), fsub(fsub(gy, fmul(sg, inv_n)), fmul(xhat, fmul(sgx, inv_n))));
}

// thread j < k
__global__ void __launch_bounds__(256)
conve_tr_bn2_bwd_kernel(const ConveTrain a, const float* __restrict__ gx, const float* __restrict__ x,
                        float* __restrict__ dh, float* g_bn2_w, float* g_bn2_b, float* g_fc_b) {
  const int j = blockIdx.x * 256 + threadIdx.x, k = a.k;
  if (j >= k) return;
  const long long G = a.Q / a.B;
  const float inv_n = __fdiv_rn(1.0f, (float)a.B), w = __ldg(a.bn2_w + j);
  float tw = 0.f, tb = 0.f, tf = 0.f;
  for (long long g = 0; g < G; ++g) {
    const long long r0 = g * a.B;
    const float mean = a.st2[(g * k + j) * 2], invstd = a.st2[(g * k + j) * 2 + 1];
    float sg = 0.f, sgx = 0.f;
    for (long long i = r0; i < r0 + a.B; ++i) {
      const long long o = i * k + j;
      const float gy = __ldg(x + o) > 0.f ? __ldg(gx + o) : 0.f;
      sg = fadd(sg, gy);
      sgx = ffma(gy, fmul(fsub(a.hpre[o], mean), invstd), sgx);
    }
    tw = fadd(tw, sgx); tb = fadd(tb, sg);
    for (long long i = r0; i < r0 + a.B; ++i) {
      const long long o = i * k + j;
      const float gy = __ldg(x + o) > 0.f ? __ldg(gx + o) : 0.f;
      float d = conve_bn_bwd(gy, fmul(fsub(a.hpre[o], mean), invstd), sg, sgx, inv_n, w, invstd);
      if (a.noise2) d = fmul(d, __ldg(a.noise2 + o));
      dh[o] = d;
      tf = fadd(tf, d);
    }
  }
  g_bn2_w[j] += tw; g_bn2_b[j] += tb; g_fc_b[j] += tf;
}

// one CTA per query: dz = d feat -> g1 = d (bn1 output) in place; per-channel (sum g1, sum g1 xhat1) partials
__global__ void __launch_bounds__(CONVE_TR_THREADS) conve_tr_bn1_bwd_part_kernel(const ConveTrain a) {
  const long long q = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int plane = (2 * a.h2 - 2) * (a.h1 - 2), F = CONVE_CH * plane;
  const long long g = q / a.B;
  for (int c = warp; c < CONVE_CH; c += CONVE_TR_THREADS / 32) {
    const float* st = a.st1 + (g * CONVE_CH + c) * 2;
    const float mean = st[0], invstd = st[1], w = __ldg(a.bn1_w + c), b = __ldg(a.bn1_b + c);
    const float nz = a.noise1 ? __ldg(a.noise1 + q * CONVE_CH + c) : 1.0f;
    float* dzc = a.dz + q * F + (long long)c * plane;
    const float* zc = a.z1 + q * F + (long long)c * plane;
    float sg = 0.f, sgx = 0.f;
    for (int p = lane; p < plane; p += 32) {
      const float xhat = fmul(fsub(__ldg(zc + p), mean), invstd);
      const float y = ffma(xhat, w, b);
      const float g1 = y > 0.f ? (a.noise1 ? fmul(dzc[p], nz) : dzc[p]) : 0.f;
      dzc[p] = g1;
      sg = fadd(sg, g1);
      sgx = ffma(g1, xhat, sgx);
    }
    sg = conve_warp_sum(sg);
    sgx = conve_warp_sum(sgx);
    if (lane == 0) { a.part1[(q * CONVE_CH + c) * 2] = sg; a.part1[(q * CONVE_CH + c) * 2 + 1] = sgx; }
  }
}

// thread c < C: red[g][c] = sum over group g's queries (ascending) of part[q][c] (pairs); gw[c] += sum_g of the
// second members, gb[c] += sum_g of the first
__global__ void __launch_bounds__(256)
conve_tr_reduce_kernel(const float* __restrict__ part, long long Q, long long B, int C, float* __restrict__ red,
                       float* gw, float* gb) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  const long long G = Q / B;
  float tw = 0.f, tb = 0.f;
  for (long long g = 0; g < G; ++g) {
    float s0 = 0.f, s1 = 0.f;
    for (long long q = g * B; q < (g + 1) * B; ++q) {
      s0 = fadd(s0, part[(q * C + c) * 2]);
      s1 = fadd(s1, part[(q * C + c) * 2 + 1]);
    }
    red[(g * C + c) * 2] = s0; red[(g * C + c) * 2 + 1] = s1;
    tb = fadd(tb, s0); tw = fadd(tw, s1);
  }
  gw[c] += tw; gb[c] += tb;
}

// out[c] += sum over q ascending of part[q][c]   (thread c < C)
__global__ void __launch_bounds__(256)
conve_tr_colsum_kernel(const float* __restrict__ part, long long Q, int C, float* out) {
  const int c = blockIdx.x * 256 + threadIdx.x;
  if (c >= C) return;
  float s = 0.f;
  for (long long q = 0; q < Q; ++q) s = fadd(s, __ldg(part + q * C + c));
  out[c] += s;
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) conve_tr_conv_bwd_kernel(const ConveTrain a) {
  __shared__ float xin[CONVE_MAX_IMAGE];
  __shared__ float wgt[CONVE_TAPS];
  __shared__ float sh[CONVE_TR_THREADS / 32];
  const long long q = blockIdx.x, g = q / a.B;
  const int tid = threadIdx.x, n0 = 2 * a.k;
  const int W = a.h1, Ho = 2 * a.h2 - 2, Wo = a.h1 - 2, plane = Ho * Wo, F = CONVE_CH * plane;
  conve_tr_conv_input(a, q, xin);
  for (int i = tid; i < CONVE_TAPS; i += CONVE_TR_THREADS) wgt[i] = __ldg(a.conv_w + i);
  // bn1 backward: g1 -> dz1 in place
  const float inv_n1 = __fdiv_rn(1.0f, fmul((float)a.B, (float)plane));
  float* dzq = a.dz + q * F;
  const float* zq = a.z1 + q * F;
  for (int o = tid; o < F; o += CONVE_TR_THREADS) {
    const int c = o / plane;
    const float* st = a.st1 + (g * CONVE_CH + c) * 2;
    const float* rd = a.red1 + (g * CONVE_CH + c) * 2;
    const float xhat = fmul(fsub(__ldg(zq + o), st[0]), st[1]);
    dzq[o] = conve_bn_bwd(dzq[o], xhat, rd[0], rd[1], inv_n1, __ldg(a.bn1_w + c), st[1]);
  }
  __syncthreads();   // dz1 of this query and xin complete
  // d conv.weight / d conv.bias of this query: one sequential chain over the output pixels per element
  for (int t = tid; t < CONVE_TAPS + CONVE_CH; t += CONVE_TR_THREADS) {
    float s = 0.f;
    if (t < CONVE_TAPS) {
      const int c = t / 9, di = (t - c * 9) / 3, dj = t - c * 9 - di * 3;
      const float* dzc = dzq + (long long)c * plane;
      for (int p = 0; p < plane; ++p) {
        const int i = p / Wo, j = p - i * Wo;
        s = ffma(dzc[p], xin[(i + di) * W + j + dj], s);
      }
      a.pw[q * CONVE_TAPS + t] = s;
    } else {
      const int c = t - CONVE_TAPS;
      const float* dzc = dzq + (long long)c * plane;
      for (int p = 0; p < plane; ++p) s = fadd(s, dzc[p]);
      a.pb[q * CONVE_CH + c] = s;
    }
  }
  // transposed conv: d xin[I][J] = sum_c sum_(di,dj) w[c][di][dj] dz1[c][I-di][J-dj], then * noise0 -> d (bn0 out)
  const float mean0 = a.st0[g * 2], invstd0 = a.st0[g * 2 + 1];
  float s0 = 0.f, s1 = 0.f;
  for (int pix = tid; pix < n0; pix += CONVE_TR_THREADS) {
    const int I = pix / W, J = pix - I * W;
    float acc = 0.f;
    for (int c = 0; c < CONVE_CH; ++c) {
      const float* dzc = dzq + (long long)c * plane;
#pragma unroll
      for (int di = 0; di < 3; ++di) {
        const int i = I - di;
        if (i < 0 || i >= Ho) continue;
#pragma unroll
        for (int dj = 0; dj < 3; ++dj) {
          const int j = J - dj;
          if (j < 0 || j >= Wo) continue;
          acc = ffma(wgt[c * 9 + di * 3 + dj], dzc[i * Wo + j], acc);
        }
      }
    }
    if (a.noise0) acc = fmul(acc, __ldg(a.noise0 + q * n0 + pix));
    a.dimg[q * n0 + pix] = acc;
    s0 = fadd(s0, acc);
    s1 = ffma(acc, fmul(fsub(a.img[q * n0 + pix], mean0), invstd0), s1);
  }
  s0 = conve_block_sum(s0, sh);
  s1 = conve_block_sum(s1, sh);
  if (tid == 0) { a.part0[q * 2] = s0; a.part0[q * 2 + 1] = s1; }
}

// bn0 backward -> the dense entity / relation gradients (one CTA per query; ids repeat: float atomics)
__global__ void __launch_bounds__(CONVE_TR_THREADS)
conve_tr_bn0_bwd_kernel(const ConveTrain a, float* gent, float* grel) {
  const long long q = blockIdx.x, g = q / a.B;
  const int k = a.k, n0 = 2 * k;
  const float mean0 = a.st0[g * 2], invstd0 = a.st0[g * 2 + 1], w = __ldg(a.bn0_w);
  const float inv_n0 = __fdiv_rn(1.0f, fmul((float)a.B, (float)n0));
  const float sg = a.red0[g * 2], sgx = a.red0[g * 2 + 1];
  const int64_t e = __ldg(a.e + q), r = __ldg(a.r + q);
  for (int pix = threadIdx.x; pix < n0; pix += CONVE_TR_THREADS) {
    const float xhat = fmul(fsub(a.img[q * n0 + pix], mean0), invstd0);
    const float d = conve_bn_bwd(a.dimg[q * n0 + pix], xhat, sg, sgx, inv_n0, w, invstd0);
    if (d == 0.f) continue;
    if (pix < k) atomicAdd(gent + e * k + pix, d);
    else atomicAdd(grel + r * k + (pix - k), d);
  }
}

// ---- launch plans of the Linear layer's backward on proj_gemm_kernel (shared with tests/emu) ---------------
// d fc.weight[k, F] += dh^T[k, Q] . feat[Q, F]   (one slice: every element receives exactly one atomic add)
inline ProjLaunch conve_plan_grad_fc_w(const float* dh, const float* feat, long long Q, long long F, int k,
                                       float* g_fc_w) {
  ProjLaunch L{};
  ProjGemm& g = L.g;
  g.A = dh; g.sAm = 1; g.sAk = k; g.Ap = nullptr;
  g.B = feat; g.sBn = 1; g.sBk = F;
  g.M = k; g.N = (int)F; g.K = (int)Q; g.klen = (int)proj_tiles(Q, PBK) * PBK;
  g.avec = 0; g.bvec = 0;
  g.C = g_fc_w; g.ldc = F;
  L.gx = proj_tiles(F, PBN); L.gy = proj_tiles(k, PBM); L.gz = 1;
  return L;
}

// dfeat[Q, F] = dh[Q, k] . fc.weight[k, F]   (stored)
inline ProjLaunch conve_plan_grad_feat(const float* dh, const float* fc_w, long long Q, long long F, int k,
                                       float* dfeat) {
  ProjLaunch L{};
  ProjGemm& g = L.g;
  g.A = dh; g.sAm = k; g.sAk = 1; g.Ap = nullptr;
  g.B = fc_w; g.sBn = 1; g.sBk = F;
  g.M = (int)Q; g.N = (int)F; g.K = k; g.klen = (int)proj_tiles(k, PBK) * PBK;
  g.avec = proj_vec_ok(dh, k, 1); g.bvec = 0;
  g.C = dfeat; g.ldc = F; g.zstride = 0; g.bias = nullptr; g.act = ACT_NONE;
  L.gx = proj_tiles(F, PBN); L.gy = proj_tiles(Q, PBM); L.gz = 1;
  return L;
}

}  // namespace kge
