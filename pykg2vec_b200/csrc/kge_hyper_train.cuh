// kge_hyper_train.cuh — HypER's trunk in TRAINING mode (pykg2vec/models/projection.py:581-606 with
// self.training == True), forward and backward, launched from kge_proj.cu (kge_hyper_train_*).
// Per query q of a group of B queries (one direction of train_step_projection), de = ent width, dr = rel width:
//     w[288] = fc1(rel[r])                     32 filters of width 9, the query's own (no activation)
//     v[de]  = bn0(ent[e]) * noise0[q, :]      bn0: batch statistics over the group's B * de values (inp_drop)
//     z1[c, j] = sum_{t<9} w[9c + t] v[j + t]  c < 32, j < Wo = de - 8 (no conv bias)
//     feat[c * Wo + j] = bn1(z1)[c, j] * noise1[q, c]   per-channel batch statistics; NO ReLU; Dropout2d
//     hpre = (feat . fc.weight^T + fc.bias) * noise2[q, :] (hidden_drop)
//     x = relu(bn2(hpre))                      per feature, over the group's B rows
// Kernels (one CTA per query unless noted) and the pieces of kge_conve_train.cuh they reuse:
//   tucker_gather_rows_kernel   relr[q] = rel[r[q]]; the filter GEMM on the tiled GEMM (hyper_plan_filters) -> filt
//   hyper_tr_gather_kernel      img[q] = ent[e[q]] (raw) + per-query (sum, centred sum of squares) of its de values
//   conve_tr_bn_stats_kernel    bn0, then bn1: the group's (mean, invstd), running statistics group after group
//   hyper_tr_conv_kernel        bn0 + noise0 + the query's 32 x 9 filters -> z1, per-query per-channel partials
//   hyper_tr_feat_kernel        feat = bn1(z1) * noise1 (elementwise)
//   (tiled GEMM) + conve_tr_fc_combine_kernel   the Linear layer in slices, + fc.bias, * noise2 -> hpre
//   conve_tr_bn2_kernel         bn2 + ReLU (on the ConveTrain view of hyper_tr_bn2_view)
// backward (gradients ACCUMULATED into dense buffers shaped like the parameters, order of kge_hyper_train_bwd):
//   conve_tr_bn2_bwd_kernel     relu mask, bn2 backward, * noise2 -> dh; d bn2.*, d fc.bias
//   (tiled GEMM)                d fc.weight += dh^T . feat (conve_plan_grad_fc_w), dfeat = dh . fc.weight
//   hyper_tr_bn1_bwd_part_kernel  * noise1 -> g1 (in place), per-query per-channel (sum g1, sum g1 xhat1)
//   conve_tr_reduce_kernel      bn1's (then bn0's) group sums -> d bn.weight, d bn.bias
//   hyper_tr_conv_bwd_kernel    bn1 backward -> dz1 (in place); dw[q, 288] (one chain over j per tap); transposed
//                               1 x 9 filter -> d v, * noise0 -> dimg; per-query bn0 partials
//   hyper_tr_bn0_bwd_kernel     bn0 backward -> grad_ent[e] (float atomics: ids repeat; the padding row skipped)
//   (tiled GEMM)                d fc1.weight += dw^T . relr (one slice), d relr = dw . fc1.weight
//   conve_tr_colsum_kernel      d fc1.bias += sum over q ascending of dw
//   hyper_tr_scatter_rel_kernel grad_rel[r] += d relr (float atomics; the padding row skipped)
//
// Canonical arithmetic of the forward: the CTA sum, warp sum, per-query partials, group statistics, normalisation
// and running-statistic update of kge_conve_train.cuh (stated at its top); the filters are kge_hyper.cuh's (one fma
// chain over dr from 0, then + fc1.bias: the same bits as the inference path's filter table); the conv is 9
// sequential fma from 0 in tap order (no bias); the Linear layer is ConvE's sliced chain.  Restated by
// tests/oracle_hyper_train bit for bit; a call over G groups equals G calls.  The backward's sums over queries run
// in a fixed order except the entity / relation scatters (float atomics).
#pragma once
#include "kge_conve_train.cuh"
#include "kge_hyper.cuh"
#include "kge_tucker.cuh"

namespace kge {

struct HyperTrain {
  const float* ent;
  const int64_t* e; const int64_t* r;
  int de, dr;
  long long Q, B;                // rows, rows per group
  long long ent_pad, rel_pad;    // padding_idx of the embeddings (-1: none): their rows get no lookup gradient
  const float* bn0_w; const float* bn0_b;
  const float* bn1_w; const float* bn1_b;
  const float* bn2_w; const float* bn2_b;
  const float* noise0;           // [Q, de] or NULL
  const float* noise1;           // [Q, 32] or NULL
  const float* noise2;           // [Q, de] or NULL
  // workspace (forward writes, backward reads; the backward's scratch follows)
  float* relr;                   // [Q, dr]     the queries' relation rows
  float* filt;                   // [Q, 288]    their filters
  float* img;                    // [Q, de]     the queries' entity rows
  float* z1;                     // [Q, F]
  float* feat;                   // [Q, F]
  float* hpre;                   // [Q, de]
  float* st0;                    // [G, 2]
  float* st1;                    // [G, 32, 2]
  float* st2;                    // [G, de, 2]
  float* part0;                  // [Q, 2]
  float* part1;                  // [Q, 32, 2]
  float* red0;                   // [G, 1, 2]
  float* red1;                   // [G, 32, 2]
  float* dh;                     // [Q, de]
  float* dz;                     // [Q, F]      d feat -> g1 -> dz1
  float* dimg;                   // [Q, de]     d (bn0 output)
  float* dw;                     // [Q, 288]    d filters
  float* drel;                   // [Q, dr]     d relation rows
};

struct HyperTrainLayout {
  long long relr, filt, img, z1, feat, partial, hpre, st0, st1, st2, part0, part1, red0, red1, dh, dz, dimg, dw, drel,
      total;
};

// float offsets of the workspace regions, each 64-float aligned (16-byte loads of the GEMM operands)
inline HyperTrainLayout hyper_train_layout(long long Q, long long B, int de, int dr) {
  const long long F = hyper_feat_width(de), S = conve_fc_slices(F), G = Q / B;
  HyperTrainLayout L{};
  long long o = 0;
  auto take = [&o](long long n) { const long long at = o; o += (n + 63) / 64 * 64; return at; };
  L.relr = take(Q * dr); L.filt = take(Q * HYPER_FILT); L.img = take(Q * de); L.z1 = take(Q * F);
  L.feat = take(Q * F); L.partial = take(S * Q * de); L.hpre = take(Q * de);
  L.st0 = take(G * 2); L.st1 = take(G * HYPER_CH * 2); L.st2 = take(G * de * 2);
  L.part0 = take(Q * 2); L.part1 = take(Q * HYPER_CH * 2);
  L.red0 = take(G * 2); L.red1 = take(G * HYPER_CH * 2);
  L.dh = take(Q * de); L.dz = take(Q * F); L.dimg = take(Q * de); L.dw = take(Q * HYPER_FILT); L.drel = take(Q * dr);
  L.total = o;
  return L;
}

// the fields conve_tr_bn2_kernel / conve_tr_bn2_bwd_kernel read (k, Q, B, bn2_*, noise2, hpre, st2), HypER's
inline ConveTrain hyper_tr_bn2_view(const HyperTrain& a) {
  ConveTrain v{};
  v.k = a.de; v.Q = a.Q; v.B = a.B;
  v.bn2_w = a.bn2_w; v.bn2_b = a.bn2_b; v.noise2 = a.noise2;
  v.hpre = a.hpre; v.st2 = a.st2;
  return v;
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) hyper_tr_gather_kernel(const HyperTrain a) {
  __shared__ float sh[CONVE_TR_THREADS / 32];
  const long long q = blockIdx.x;
  const int de = a.de, tid = threadIdx.x;
  const float* er = a.ent + __ldg(a.e + q) * (long long)de;
  float* out = a.img + q * de;
  float s = 0.f;
  for (int i = tid; i < de; i += CONVE_TR_THREADS) {
    const float v = __ldg(er + i);
    out[i] = v;
    s = fadd(s, v);
  }
  s = conve_block_sum(s, sh);
  const float m = __fdiv_rn(s, (float)de);
  float m2 = 0.f;
  for (int i = tid; i < de; i += CONVE_TR_THREADS) {   // this thread's own elements: no barrier needed
    const float d = fsub(out[i], m);
    m2 = ffma(d, d, m2);
  }
  m2 = conve_block_sum(m2, sh);
  if (tid == 0) { a.part0[q * 2] = s; a.part0[q * 2 + 1] = m2; }
}

// bn0 + noise0 of query q into shared memory, and its 288 filter taps: the conv input of the forward and backward
KGE_DEV void hyper_tr_conv_input(const HyperTrain& a, long long q, float* xin, float* wgt) {
  const int de = a.de;
  const long long g = q / a.B;
  const float mean = a.st0[g * 2], invstd = a.st0[g * 2 + 1], w = __ldg(a.bn0_w), b = __ldg(a.bn0_b);
  for (int i = threadIdx.x; i < de; i += CONVE_TR_THREADS) {
    float v = conve_bn_apply(a.img[q * de + i], mean, invstd, w, b);
    if (a.noise0) v = fmul(v, __ldg(a.noise0 + q * de + i));
    xin[i] = v;
  }
  for (int i = threadIdx.x; i < HYPER_FILT; i += CONVE_TR_THREADS) wgt[i] = a.filt[q * HYPER_FILT + i];
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) hyper_tr_conv_kernel(const HyperTrain a) {
  __shared__ float xin[HYPER_MAX_DE];
  __shared__ float wgt[HYPER_FILT];
  const long long q = blockIdx.x;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int Wo = a.de - HYPER_FW + 1, F = HYPER_CH * Wo;
  hyper_tr_conv_input(a, q, xin, wgt);
  __syncthreads();
  float* out = a.z1 + q * F;
  for (int o = tid; o < F; o += CONVE_TR_THREADS) {
    const int c = o / Wo, j = o - c * Wo;
    float acc = 0.f;
#pragma unroll
    for (int t = 0; t < HYPER_FW; ++t) acc = ffma(wgt[c * HYPER_FW + t], xin[j + t], acc);
    out[o] = acc;
  }
  __syncthreads();   // z1 of this query is complete (global writes of the CTA are visible after the barrier)
  for (int c = warp; c < HYPER_CH; c += CONVE_TR_THREADS / 32) {
    const float* zc = out + c * Wo;
    float s = 0.f;
    for (int p = lane; p < Wo; p += 32) s = fadd(s, zc[p]);
    s = conve_warp_sum(s);
    const float m = __fdiv_rn(s, (float)Wo);
    float m2 = 0.f;
    for (int p = lane; p < Wo; p += 32) {
      const float d = fsub(zc[p], m);
      m2 = ffma(d, d, m2);
    }
    m2 = conve_warp_sum(m2);
    if (lane == 0) { a.part1[(q * HYPER_CH + c) * 2] = s; a.part1[(q * HYPER_CH + c) * 2 + 1] = m2; }
  }
}

__global__ void __launch_bounds__(256) hyper_tr_feat_kernel(const HyperTrain a, long long F, int Wo) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.Q * F) return;
  const long long q = i / F;
  const int c = (int)((i - q * F) / Wo);
  const float* st = a.st1 + ((q / a.B) * HYPER_CH + c) * 2;
  float v = conve_bn_apply(__ldg(a.z1 + i), st[0], st[1], __ldg(a.bn1_w + c), __ldg(a.bn1_b + c));
  if (a.noise1) v = fmul(v, __ldg(a.noise1 + q * HYPER_CH + c));
  a.feat[i] = v;
}

// ---- backward ------------------------------------------------------------------------------------------------

// one CTA per query: dz = d feat -> g1 = d (bn1 output) = d feat * noise1 in place; per-channel (sum g1, sum g1 xhat1)
__global__ void __launch_bounds__(CONVE_TR_THREADS) hyper_tr_bn1_bwd_part_kernel(const HyperTrain a) {
  const long long q = blockIdx.x, g = q / a.B;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int Wo = a.de - HYPER_FW + 1, F = HYPER_CH * Wo;
  for (int c = warp; c < HYPER_CH; c += CONVE_TR_THREADS / 32) {
    const float* st = a.st1 + (g * HYPER_CH + c) * 2;
    const float mean = st[0], invstd = st[1];
    const float nz = a.noise1 ? __ldg(a.noise1 + q * HYPER_CH + c) : 1.0f;
    float* dzc = a.dz + q * F + (long long)c * Wo;
    const float* zc = a.z1 + q * F + (long long)c * Wo;
    float sg = 0.f, sgx = 0.f;
    for (int p = lane; p < Wo; p += 32) {
      const float xhat = fmul(fsub(__ldg(zc + p), mean), invstd);
      const float g1 = a.noise1 ? fmul(dzc[p], nz) : dzc[p];
      dzc[p] = g1;
      sg = fadd(sg, g1);
      sgx = ffma(g1, xhat, sgx);
    }
    sg = conve_warp_sum(sg);
    sgx = conve_warp_sum(sgx);
    if (lane == 0) { a.part1[(q * HYPER_CH + c) * 2] = sg; a.part1[(q * HYPER_CH + c) * 2 + 1] = sgx; }
  }
}

__global__ void __launch_bounds__(CONVE_TR_THREADS) hyper_tr_conv_bwd_kernel(const HyperTrain a) {
  __shared__ float xin[HYPER_MAX_DE];
  __shared__ float wgt[HYPER_FILT];
  __shared__ float sh[CONVE_TR_THREADS / 32];
  const long long q = blockIdx.x, g = q / a.B;
  const int tid = threadIdx.x, de = a.de, Wo = de - HYPER_FW + 1, F = HYPER_CH * Wo;
  hyper_tr_conv_input(a, q, xin, wgt);
  // bn1 backward: g1 -> dz1 in place
  const float inv_n1 = __fdiv_rn(1.0f, fmul((float)a.B, (float)Wo));
  float* dzq = a.dz + q * F;
  const float* zq = a.z1 + q * F;
  for (int o = tid; o < F; o += CONVE_TR_THREADS) {
    const int c = o / Wo;
    const float* st = a.st1 + (g * HYPER_CH + c) * 2;
    const float* rd = a.red1 + (g * HYPER_CH + c) * 2;
    const float xhat = fmul(fsub(__ldg(zq + o), st[0]), st[1]);
    dzq[o] = conve_bn_bwd(dzq[o], xhat, rd[0], rd[1], inv_n1, __ldg(a.bn1_w + c), st[1]);
  }
  __syncthreads();   // dz1 of this query, xin and the filters complete
  // d filters of this query: one sequential chain over the output positions per tap
  for (int t = tid; t < HYPER_FILT; t += CONVE_TR_THREADS) {
    const int c = t / HYPER_FW, tap = t - c * HYPER_FW;
    const float* dzc = dzq + (long long)c * Wo;
    float s = 0.f;
    for (int j = 0; j < Wo; ++j) s = ffma(dzc[j], xin[j + tap], s);
    a.dw[q * HYPER_FILT + t] = s;
  }
  // transposed filter: d v[i] = sum_c sum_t w[c][t] dz1[c][i - t], then * noise0 -> d (bn0 output)
  const float mean0 = a.st0[g * 2], invstd0 = a.st0[g * 2 + 1];
  float s0 = 0.f, s1 = 0.f;
  for (int i = tid; i < de; i += CONVE_TR_THREADS) {
    float acc = 0.f;
    for (int c = 0; c < HYPER_CH; ++c) {
      const float* dzc = dzq + (long long)c * Wo;
#pragma unroll
      for (int t = 0; t < HYPER_FW; ++t) {
        const int j = i - t;
        if (j >= 0 && j < Wo) acc = ffma(wgt[c * HYPER_FW + t], dzc[j], acc);
      }
    }
    if (a.noise0) acc = fmul(acc, __ldg(a.noise0 + q * de + i));
    a.dimg[q * de + i] = acc;
    s0 = fadd(s0, acc);
    s1 = ffma(acc, fmul(fsub(a.img[q * de + i], mean0), invstd0), s1);
  }
  s0 = conve_block_sum(s0, sh);
  s1 = conve_block_sum(s1, sh);
  if (tid == 0) { a.part0[q * 2] = s0; a.part0[q * 2 + 1] = s1; }
}

// bn0 backward -> the dense entity gradient (one CTA per query; ids repeat: float atomics; the padding row skipped)
__global__ void __launch_bounds__(CONVE_TR_THREADS) hyper_tr_bn0_bwd_kernel(const HyperTrain a, float* gent) {
  const long long q = blockIdx.x, g = q / a.B;
  const int64_t e = __ldg(a.e + q);
  if (e == a.ent_pad) return;
  const int de = a.de;
  const float mean0 = a.st0[g * 2], invstd0 = a.st0[g * 2 + 1], w = __ldg(a.bn0_w);
  const float inv_n0 = __fdiv_rn(1.0f, fmul((float)a.B, (float)de));
  const float sg = a.red0[g * 2], sgx = a.red0[g * 2 + 1];
  for (int i = threadIdx.x; i < de; i += CONVE_TR_THREADS) {
    const float xhat = fmul(fsub(a.img[q * de + i], mean0), invstd0);
    const float d = conve_bn_bwd(a.dimg[q * de + i], xhat, sg, sgx, inv_n0, w, invstd0);
    if (d != 0.f) atomicAdd(gent + e * de + i, d);
  }
}

// grel[r[q], :] += drel[q, :] except for the padding row (float atomics: ids repeat)
__global__ void __launch_bounds__(256)
hyper_tr_scatter_rel_kernel(const float* __restrict__ drel, const int64_t* __restrict__ r, long long Q, int dr,
                            long long pad, float* __restrict__ grel) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= Q * dr) return;
  const long long q = i / dr;
  const int64_t id = __ldg(r + q);
  if (id != pad) atomicAdd(grel + id * dr + (i - q * dr), __ldg(drel + i));
}

}  // namespace kge
