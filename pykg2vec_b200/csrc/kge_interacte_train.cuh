// kge_interacte_train.cuh — InteractE's trunk in TRAINING mode (pykg2vec/models/projection.py:425-442 with
// self.training == True), forward and backward, launched from kge_proj.cu (kge_interacte_train_*).
// Per query q of a group of B queries (one direction of train_step_projection), with P images of H = 2 *
// reshape_width rows and W = reshape_height columns, HW = H * W = 2k, pad = ks / 2, C1 = P * F channels:
//     comb = [ent[e] ; rel[r]]                                 2k values
//     img[p][pix] = comb[perm[p][pix]]                         p < P (the chequer permutation)
//     v[p] = bn0_p(img[p]) * noise0[q, p, :]                   bn0: per image channel p, over the group's B * HW values
//     z1[p*F+f][i][j] = sum_{u,v<ks} filt[f][u][v] * v[p][(i+u-pad) mod H][(j+v-pad) mod W]    (no bias)
//     feat = relu(bn1(z1)) * noise1[q, c]                      per-channel statistics over B * HW; Dropout2d
//     hpre = (feat . fc.weight^T + fc.bias) * noise2[q, :]     (hidden_drop)
//     x = relu(bn2(hpre))                                      per feature, over the group's B rows
// Kernels (one CTA per query unless noted) and the pieces of kge_conve_train.cuh they reuse:
//   interacte_tr_gather_kernel   img[q] = the P permuted images (raw) + per-query per-image (sum, centred sum of
//                                squares) over its HW values (CTA sums, pixel order)
//   conve_tr_bn_stats_kernel     bn0 (P channels), then bn1 (C1 channels): (mean, invstd), running statistics
//   interacte_tr_conv_kernel     bn0 + noise0 into P circularly padded images in shared memory, the circular conv
//                                (kge_interacte.cuh's INTERACTE_FB register blocking) -> z1; per-channel partials
//   interacte_tr_feat_kernel     feat = relu(bn1(z1)) * noise1 (elementwise)
//   (tiled GEMM) + conve_tr_fc_combine_kernel   the Linear layer in slices, + fc.bias, * noise2 -> hpre
//   conve_tr_bn2_kernel          bn2 + ReLU (on the ConveTrain view of interacte_tr_bn2_view)
// backward (gradients ACCUMULATED into dense buffers shaped like the parameters, order of kge_interacte_train_bwd):
//   conve_tr_bn2_bwd_kernel      relu mask, bn2 backward, * noise2 -> dh; d bn2.*, d fc.bias
//   (tiled GEMM)                 d fc.weight += dh^T . feat, THEN d feat = dh . fc.weight into feat's buffer
//   interacte_tr_bn1_bwd_part_kernel  relu mask (recomputed from z1) * noise1 -> g1 (in place), per-channel partials
//   conve_tr_reduce_kernel       bn1's (then bn0's) group sums -> d bn.weight, d bn.bias
//   interacte_tr_conv_bwd_kernel bn1 backward -> dz1 (in place); per-query d conv_filt [F, ks*ks] (one chain over
//                                p, then the HW positions, per tap); the transposed circular conv -> d v, * noise0
//                                -> dimg; per-query per-image bn0 partials
//   conve_tr_colsum_kernel       d conv_filt += sum over q ascending of the per-query partials
//   interacte_tr_bn0_bwd_kernel  bn0 backward, un-permute (d comb[c] = sum over p ascending of d img[p] at the pixel
//                                perm[p] sends c to) -> grad_ent[e] / grad_rel[r] (float atomics: ids repeat)
//
// Canonical arithmetic of the forward: the CTA sum, warp sum, per-query partials, group statistics, normalisation
// and running-statistic update of kge_conve_train.cuh (stated at its top), bn0's partials one CTA sum per image in
// pixel order; the conv is kge_interacte.cuh's (ks * ks sequential fma from 0, row u then column v, no bias); the
// Linear layer is ConvE's sliced chain.  Restated by tests/oracle_interacte_train bit for bit; a call over G groups
// equals G calls.  The backward's sums over queries run in a fixed order except the entity / relation scatter.
#pragma once
#include "kge_conve_train.cuh"
#include "kge_interacte.cuh"

namespace kge {

struct InteracteTrain {
  const float* ent; const float* rel;
  const int64_t* perm;           // [P, HW], each row a permutation of 0 .. HW-1
  const int64_t* e; const int64_t* r;
  int P, F, ks, H, W;
  long long Q, B;                // rows, rows per group
  const float* bn0_w; const float* bn0_b;
  const float* filt;             // [F, 1, ks, ks]
  const float* bn1_w; const float* bn1_b;
  const float* bn2_w; const float* bn2_b;
  const float* noise0;           // [Q, P * HW] or NULL
  const float* noise1;           // [Q, C1] or NULL
  const float* noise2;           // [Q, k] or NULL
  // workspace (forward writes, backward reads; the backward's scratch follows)
  float* img;                    // [Q, P, HW]  the permuted images (raw)
  float* z1;                     // [Q, Fw]
  float* feat;                   // [Q, Fw]     feat; in the backward d feat -> g1 -> dz1
  float* hpre;                   // [Q, k]
  float* st0;                    // [G, P, 2]
  float* st1;                    // [G, C1, 2]
  float* st2;                    // [G, k, 2]
  float* part0;                  // [Q, P, 2]
  float* part1;                  // [Q, C1, 2]
  float* red0;                   // [G, P, 2]
  float* red1;                   // [G, C1, 2]
  float* dh;                     // [Q, k]
  float* dimg;                   // [Q, P, HW]  d (bn0 output)
  float* pw;                     // [Q, F * ks * ks]  per-query d conv_filt
};

struct InteracteTrainLayout {
  long long img, z1, feat, partial, hpre, st0, st1, st2, part0, part1, red0, red1, dh, dimg, pw, total;
};

// float offsets of the workspace regions, each 64-float aligned (16-byte loads of the GEMM operands).  Two
// full-width [Q, Fw] arrays (z1 and feat / d feat); the rest is O(Q * (k * slices + HW * P + F * ks^2)).
inline InteracteTrainLayout interacte_train_layout(long long Q, long long B, int P, int F, int ks, int H, int W) {
  const long long HW = (long long)H * W, k = HW / 2, C1 = (long long)P * F, Fw = C1 * HW;
  const long long S = conve_fc_slices(Fw), G = Q / B;
  InteracteTrainLayout L{};
  long long o = 0;
  auto take = [&o](long long n) { const long long at = o; o += (n + 63) / 64 * 64; return at; };
  L.img = take(Q * P * HW); L.z1 = take(Q * Fw); L.feat = take(Q * Fw); L.partial = take(S * Q * k);
  L.hpre = take(Q * k);
  L.st0 = take(G * P * 2); L.st1 = take(G * C1 * 2); L.st2 = take(G * k * 2);
  L.part0 = take(Q * P * 2); L.part1 = take(Q * C1 * 2);
  L.red0 = take(G * P * 2); L.red1 = take(G * C1 * 2);
  L.dh = take(Q * k); L.dimg = take(Q * P * HW); L.pw = take(Q * F * ks * ks);
  L.total = o;
  return L;
}

// Shared memory of the conv kernels, in floats: the filter bank transposed to [ks*ks][Fpad] (zero columns f >= F),
// then the P circularly padded bn0 outputs [(H + 2 pad)][(W + 2 pad)] (interacte_smem without the bn1 folds).
struct InteracteTrainSmem { long long wt, img, total; };

__host__ __device__ inline InteracteTrainSmem interacte_train_smem(int P, int F, int ks, int H, int W) {
  const long long Fp = interacte_fpad(F), pad = ks / 2;
  InteracteTrainSmem S;
  S.wt = 0;
  S.img = (long long)ks * ks * Fp;
  S.total = S.img + (long long)P * (H + 2 * pad) * (W + 2 * pad);
  return S;
}

// the fields conve_tr_bn2_kernel / conve_tr_bn2_bwd_kernel read (k, Q, B, bn2_*, noise2, hpre, st2), InteractE's
inline ConveTrain interacte_tr_bn2_view(const InteracteTrain& a) {
  ConveTrain v{};
  v.k = a.H * a.W / 2; v.Q = a.Q; v.B = a.B;
  v.bn2_w = a.bn2_w; v.bn2_b = a.bn2_b; v.noise2 = a.noise2;
  v.hpre = a.hpre; v.st2 = a.st2;
  return v;
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) interacte_tr_gather_kernel(const InteracteTrain a) {
  __shared__ float sh[CONVE_TR_THREADS / 32];
  const long long q = blockIdx.x;
  const int HW = a.H * a.W, k = HW / 2, tid = threadIdx.x;
  const float* er = a.ent + __ldg(a.e + q) * (long long)k;
  const float* rr = a.rel + __ldg(a.r + q) * (long long)k;
  for (int p = 0; p < a.P; ++p) {
    const int64_t* pm = a.perm + (long long)p * HW;
    float* out = a.img + (q * a.P + p) * HW;
    float s = 0.f;
    for (int i = tid; i < HW; i += CONVE_TR_THREADS) {
      const int64_t c = __ldg(pm + i);
      const float v = c < k ? __ldg(er + c) : __ldg(rr + (c - k));
      out[i] = v;
      s = fadd(s, v);
    }
    s = conve_block_sum(s, sh);
    const float m = __fdiv_rn(s, (float)HW);
    float m2 = 0.f;
    for (int i = tid; i < HW; i += CONVE_TR_THREADS) {   // this thread's own elements: no barrier needed
      const float d = fsub(out[i], m);
      m2 = ffma(d, d, m2);
    }
    m2 = conve_block_sum(m2, sh);
    if (tid == 0) { a.part0[(q * a.P + p) * 2] = s; a.part0[(q * a.P + p) * 2 + 1] = m2; }
  }
}

// the conv input of query q in shared memory: the transposed filter bank, and bn0 + noise0 of the P images,
// circularly padded (pad <= H and pad <= W, so one wrap suffices).  No barrier inside.
KGE_DEV void interacte_tr_conv_input(const InteracteTrain& a, long long q, float* wt, float* pim) {
  const int P = a.P, F = a.F, ks = a.ks, H = a.H, W = a.W, pad = ks / 2;
  const int Fp = interacte_fpad(F), taps = ks * ks, HW = H * W;
  const int Hp = H + 2 * pad, Wp = W + 2 * pad, plane = Hp * Wp;
  const long long g = q / a.B;
  for (int i = threadIdx.x; i < taps * Fp; i += CONVE_TR_THREADS) {
    const int t = i / Fp, f = i - t * Fp;
    wt[i] = f < F ? __ldg(a.filt + (long long)f * taps + t) : 0.f;
  }
  for (int i = threadIdx.x; i < P * plane; i += CONVE_TR_THREADS) {
    const int pp = i / plane, rem = i - pp * plane, pi = rem / Wp, pj = rem - pi * Wp;
    int si = pi - pad, sj = pj - pad;
    si += si < 0 ? H : (si >= H ? -H : 0);
    sj += sj < 0 ? W : (sj >= W ? -W : 0);
    const int pix = si * W + sj;
    const float* st = a.st0 + (g * P + pp) * 2;
    float v = conve_bn_apply(a.img[(q * P + pp) * HW + pix], st[0], st[1], __ldg(a.bn0_w + pp), __ldg(a.bn0_b + pp));
    if (a.noise0) v = fmul(v, __ldg(a.noise0 + (q * P + pp) * HW + pix));
    pim[i] = v;
  }
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) interacte_tr_conv_kernel(const InteracteTrain a) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else   // host emulation (tests/emu): __shared__ is a function-local static there, so it needs a fixed size
  __shared__ float4 smem_f4[INTERACTE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const long long q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int P = a.P, F = a.F, ks = a.ks, H = a.H, W = a.W, pad = ks / 2;
  const int Fp = interacte_fpad(F), HW = H * W, C1 = P * F;
  const int Hp = H + 2 * pad, Wp = W + 2 * pad, plane = Hp * Wp;
  const InteracteTrainSmem S = interacte_train_smem(P, F, ks, H, W);
  float* wt = sm + S.wt;
  float* pim = sm + S.img;
  interacte_tr_conv_input(a, q, wt, pim);
  __syncthreads();
  const int G = Fp / INTERACTE_FB, items = P * G * HW;
  float* out = a.z1 + q * C1 * HW;
  for (int it = tid; it < items; it += CONVE_TR_THREADS) {
    const int pg = it / HW, pix = it - pg * HW, pp = pg / G, gi = pg - pp * G;
    const int i = pix / W, j = pix - i * W;
    const float* ip = pim + pp * plane + i * Wp + j;
    const float* wp = wt + gi * INTERACTE_FB;
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
    const int f0 = gi * INTERACTE_FB;
#pragma unroll
    for (int b = 0; b < INTERACTE_FB; ++b)
      if (f0 + b < F) out[(long long)(pp * F + f0 + b) * HW + pix] = acc[b];
  }
  __syncthreads();   // z1 of this query is complete (global writes of the CTA are visible after the barrier)
  for (int c = warp; c < C1; c += CONVE_TR_THREADS / 32) {
    const float* zc = out + (long long)c * HW;
    float s = 0.f;
    for (int p = lane; p < HW; p += 32) s = fadd(s, zc[p]);
    s = conve_warp_sum(s);
    const float m = __fdiv_rn(s, (float)HW);
    float m2 = 0.f;
    for (int p = lane; p < HW; p += 32) {
      const float d = fsub(zc[p], m);
      m2 = ffma(d, d, m2);
    }
    m2 = conve_warp_sum(m2);
    if (lane == 0) { a.part1[(q * C1 + c) * 2] = s; a.part1[(q * C1 + c) * 2 + 1] = m2; }
  }
}

__global__ void __launch_bounds__(256) interacte_tr_feat_kernel(const InteracteTrain a, long long Fw, int HW) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.Q * Fw) return;
  const long long q = i / Fw;
  const int C1 = a.P * a.F, c = (int)((i - q * Fw) / HW);
  const float* st = a.st1 + ((q / a.B) * C1 + c) * 2;
  float v = fmaxf(conve_bn_apply(__ldg(a.z1 + i), st[0], st[1], __ldg(a.bn1_w + c), __ldg(a.bn1_b + c)), 0.f);
  if (a.noise1) v = fmul(v, __ldg(a.noise1 + q * C1 + c));
  a.feat[i] = v;
}

// ---- backward ------------------------------------------------------------------------------------------------

// one CTA per query: feat's buffer holds d feat -> g1 = d (bn1 output) in place, the relu mask recomputed from z1;
// per-channel (sum g1, sum g1 xhat1) partials
__global__ void __launch_bounds__(CONVE_TR_THREADS) interacte_tr_bn1_bwd_part_kernel(const InteracteTrain a) {
  const long long q = blockIdx.x, g = q / a.B;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int HW = a.H * a.W, C1 = a.P * a.F;
  const long long Fw = (long long)C1 * HW;
  for (int c = warp; c < C1; c += CONVE_TR_THREADS / 32) {
    const float* st = a.st1 + (g * C1 + c) * 2;
    const float mean = st[0], invstd = st[1], w = __ldg(a.bn1_w + c), b = __ldg(a.bn1_b + c);
    const float nz = a.noise1 ? __ldg(a.noise1 + q * C1 + c) : 1.0f;
    float* dzc = a.feat + q * Fw + (long long)c * HW;
    const float* zc = a.z1 + q * Fw + (long long)c * HW;
    float sg = 0.f, sgx = 0.f;
    for (int p = lane; p < HW; p += 32) {
      const float xhat = fmul(fsub(__ldg(zc + p), mean), invstd);
      const float y = ffma(xhat, w, b);
      const float g1 = y > 0.f ? (a.noise1 ? fmul(dzc[p], nz) : dzc[p]) : 0.f;
      dzc[p] = g1;
      sg = fadd(sg, g1);
      sgx = ffma(g1, xhat, sgx);
    }
    sg = conve_warp_sum(sg);
    sgx = conve_warp_sum(sgx);
    if (lane == 0) { a.part1[(q * C1 + c) * 2] = sg; a.part1[(q * C1 + c) * 2 + 1] = sgx; }
  }
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) interacte_tr_conv_bwd_kernel(const InteracteTrain a) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[INTERACTE_SMEM_MAX / 16];
#endif
  __shared__ float sh[CONVE_TR_THREADS / 32];
  float* sm = reinterpret_cast<float*>(smem_f4);
  const long long q = blockIdx.x, g = q / a.B;
  const int tid = threadIdx.x;
  const int P = a.P, F = a.F, ks = a.ks, H = a.H, W = a.W, pad = ks / 2;
  const int Fp = interacte_fpad(F), HW = H * W, C1 = P * F, taps = ks * ks;
  const int Wp = W + 2 * pad, plane = (H + 2 * pad) * Wp;
  const InteracteTrainSmem S = interacte_train_smem(P, F, ks, H, W);
  float* wt = sm + S.wt;
  float* pim = sm + S.img;
  interacte_tr_conv_input(a, q, wt, pim);
  // bn1 backward: g1 -> dz1 in place
  const float inv_n1 = __fdiv_rn(1.0f, fmul((float)a.B, (float)HW));
  float* dzq = a.feat + q * C1 * HW;
  const float* zq = a.z1 + q * C1 * HW;
  for (int o = tid; o < C1 * HW; o += CONVE_TR_THREADS) {
    const int c = o / HW;
    const float* st = a.st1 + (g * C1 + c) * 2;
    const float* rd = a.red1 + (g * C1 + c) * 2;
    const float xhat = fmul(fsub(__ldg(zq + o), st[0]), st[1]);
    dzq[o] = conve_bn_bwd(dzq[o], xhat, rd[0], rd[1], inv_n1, __ldg(a.bn1_w + c), st[1]);
  }
  __syncthreads();   // dz1 of this query, the padded images and the filters complete
  // d conv_filt of this query: per (filter, tap) one sequential chain over the images p, then the positions
  for (int t = tid; t < F * taps; t += CONVE_TR_THREADS) {
    const int f = t / taps, tap = t - f * taps, u = tap / ks, v = tap - u * ks;
    float s = 0.f;
    for (int p = 0; p < P; ++p) {
      const float* dzc = dzq + (long long)(p * F + f) * HW;
      const float* ip = pim + p * plane + u * Wp + v;
      for (int i = 0; i < H; ++i)
        for (int j = 0; j < W; ++j) s = ffma(dzc[i * W + j], ip[i * Wp + j], s);
    }
    a.pw[q * F * taps + t] = s;
  }
  // transposed circular conv: d v[p][I][J] = sum_f sum_(u,v) filt[f][u][v] dz1[p*F+f][(I-u+pad) mod H][(J-v+pad) mod W]
  for (int it = tid; it < P * HW; it += CONVE_TR_THREADS) {
    const int p = it / HW, pix = it - p * HW, I = pix / W, J = pix - I * W;
    float acc = 0.f;
    for (int f = 0; f < F; ++f) {
      const float* dzc = dzq + (long long)(p * F + f) * HW;
      for (int u = 0; u < ks; ++u) {
        int i = I - u + pad;
        i += i < 0 ? H : (i >= H ? -H : 0);
        const float* drow = dzc + i * W;
        const float* wrow = wt + u * ks * Fp + f;
        for (int v = 0; v < ks; ++v) {
          int j = J - v + pad;
          j += j < 0 ? W : (j >= W ? -W : 0);
          acc = ffma(wrow[v * Fp], drow[j], acc);
        }
      }
    }
    if (a.noise0) acc = fmul(acc, __ldg(a.noise0 + (q * P + p) * HW + pix));
    a.dimg[(q * P + p) * HW + pix] = acc;
  }
  __syncthreads();   // dimg of this query complete
  // per-image bn0 partials (sum g, sum g xhat0)
  for (int p = 0; p < P; ++p) {
    const float* st = a.st0 + (g * P + p) * 2;
    const float* dp = a.dimg + (q * P + p) * HW;
    const float* ip = a.img + (q * P + p) * HW;
    float s0 = 0.f, s1 = 0.f;
    for (int pix = tid; pix < HW; pix += CONVE_TR_THREADS) {
      const float d = dp[pix];
      s0 = fadd(s0, d);
      s1 = ffma(d, fmul(fsub(ip[pix], st[0]), st[1]), s1);
    }
    s0 = conve_block_sum(s0, sh);
    s1 = conve_block_sum(s1, sh);
    if (tid == 0) { a.part0[(q * P + p) * 2] = s0; a.part0[(q * P + p) * 2 + 1] = s1; }
  }
}

// bn0 backward and the un-permute -> the dense entity / relation gradients (one CTA per query; ids repeat: float
// atomics).  Shared memory: the inverse permutations [P][HW] (int).
__global__ void __launch_bounds__(CONVE_TR_THREADS)
interacte_tr_bn0_bwd_kernel(const InteracteTrain a, float* gent, float* grel) {
#ifdef __CUDACC__
  extern __shared__ int inv_perm[];
#else
  __shared__ int inv_perm[INTERACTE_SMEM_MAX / 4];
#endif
  const long long q = blockIdx.x, g = q / a.B;
  const int P = a.P, HW = a.H * a.W, k = HW / 2;
  for (int i = threadIdx.x; i < P * HW; i += CONVE_TR_THREADS) {
    const int p = i / HW, pix = i - p * HW;
    inv_perm[p * HW + (int)__ldg(a.perm + i)] = pix;
  }
  __syncthreads();
  const float inv_n0 = __fdiv_rn(1.0f, fmul((float)a.B, (float)HW));
  const int64_t e = __ldg(a.e + q), r = __ldg(a.r + q);
  for (int c = threadIdx.x; c < HW; c += CONVE_TR_THREADS) {
    float d = 0.f;
    for (int p = 0; p < P; ++p) {
      const float* st = a.st0 + (g * P + p) * 2;
      const float* rd = a.red0 + (g * P + p) * 2;
      const long long at = (q * P + p) * HW + inv_perm[p * HW + c];
      const float xhat = fmul(fsub(a.img[at], st[0]), st[1]);
      d = fadd(d, conve_bn_bwd(a.dimg[at], xhat, rd[0], rd[1], inv_n0, __ldg(a.bn0_w + p), st[1]));
    }
    if (d == 0.f) continue;
    if (c < k) atomicAdd(gent + e * k + c, d);
    else atomicAdd(grel + r * k + (c - k), d);
  }
}

}  // namespace kge
