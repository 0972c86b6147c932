// kge_acre_train.cuh — AcrE's trunk in TRAINING mode (pykg2vec/models/projection.py:706-734 with
// self.training == True), forward and backward, launched from kge_proj.cu (kge_acre_train_*).
// Per query q of a group of B queries (one direction of train_step_projection), C = in_channels, PIX = 400:
//     img = [ent[e] ; rel[r]]                              400 values, read as 20 x 20
//     v = bn0(img) * noise0[q, :]                          bn0: one channel over the group's B * 400 values
//     serial:   a1 = conv1(v), a2 = conv2(a1), y = conv3(a2) + v        1 -> C -> C -> C, v on every channel
//     parallel: gate[c] = [v ; conv1(v)[c] ; conv2(v)[c] ; conv3(v)[c]], y[c] = W_gate_e(gate[c])
//     feat = relu(bn1(y)) * noise1[q, c]                   per-channel statistics over B * 400; Dropout2d
//     hpre = (feat . fc.weight^T + fc.bias) * noise2[q, :]
//     x = relu(bn2(hpre))                                  per feature, over the group's B rows
// Kernels (one CTA per query unless noted) and the pieces of kge_conve_train.cuh / kge_acre.cuh they reuse:
//   conve_tr_gather_kernel       img (raw) + per-query bn0 partials (k = 200: its 2k-value image is AcrE's)
//   conve_tr_bn_stats_kernel     bn0 (1 channel), then bn1 (C channels): (mean, invstd), running statistics
//   acre_tr_serial_kernel        bn0 + noise0 -> v in shared memory, then conv1 -> a1, conv2 -> a2, conv3 + v -> y,
//                                each layer on kge_acre.cuh's acre_stage_bank / acre_conv_layer (4 pixels x 8
//                                channels per thread); a1 and a2 are kept for the backward
//   acre_tr_gate_kernel          (parallel) v, then the gate rows [Q*C, 1600]; W_gate_e on the tiled GEMM -> y
//   acre_tr_bn1_part_kernel      per-query per-channel (sum, centred sum of squares) of y (warp sums)
//   acre_tr_feat_kernel          feat = relu(bn1(y)) * noise1 (elementwise)
//   (tiled GEMM) + conve_tr_fc_combine_kernel   the Linear layer in slices, + fc.bias, * noise2 -> hpre
//   conve_tr_bn2_kernel          bn2 + ReLU (on the ConveTrain view of acre_tr_view)
// backward (gradients ACCUMULATED into dense buffers shaped like the parameters, order of kge_acre_train_bwd):
//   conve_tr_bn2_bwd_kernel      relu mask, bn2 backward, * noise2 -> dh; d bn2.*, d fc.bias
//   (tiled GEMM)                 d fc.weight += dh^T . feat, THEN d feat = dh . fc.weight into feat's buffer
//   acre_tr_bn1_bwd_part_kernel  relu mask (recomputed from y) * noise1 -> g1 (in place), per-channel partials
//   conve_tr_reduce_kernel       bn1's (later bn0's) group sums -> d bn.weight, d bn.bias
//   acre_tr_bn1_bwd_kernel       bn1 backward -> dy (in place, elementwise)
//   serial:   acre_tr_serial_bwd_kernel   per layer 3, 2, 1: the per-query weight / bias gradients (acre_tr_wgrad,
//                                         blocked 8 output x 4 input channels per thread, pixels over 4 lanes),
//                                         then the transposed conv (acre_conv_layer on a tap-flipped, transposed
//                                         bank); d v = d a0 + sum_c dy[c]; * noise0 -> dimg
//   parallel: (tiled GEMM) d W_gate_e.weight += dy^T . gate, THEN d gate = dy . W_gate_e.weight into gate's buffer;
//             conve_tr_colsum_kernel d W_gate_e.bias; acre_tr_gate_bwd_kernel the three convs' per-query weight /
//             bias gradients, d v = sum_c d gate[c][0] + the transposed convs; * noise0 -> dimg
//   conve_tr_colsum_kernel       d conv*.weight / bias += sum over q ascending of the per-query partials
//   acre_tr_bn0_part_kernel      per-query bn0 partials (sum g, sum g xhat0) of dimg (CTA sums)
//   conve_tr_bn0_bwd_kernel      bn0 backward -> grad_ent[e] (first 200) / grad_rel[r] (float atomics: ids repeat)
//
// Canonical arithmetic of the forward: the CTA sum, warp sum, per-query partials, group statistics, normalisation
// and running-statistic update of kge_conve_train.cuh (stated at its top; bn1's partials are one warp sum per
// channel over the 400 pixels in order); the convs are kge_acre.cuh's (one fma chain from 0 in tap-major order,
// padding taps skipped, + bias as a separate add); the serial residual is a separate add; W_gate_e is the tiled
// GEMM's chain + its bias; dropout is fmul by the noise; the Linear layer is ConvE's sliced chain.  A call over G
// groups equals G calls.  The backward's sums over queries run in a fixed order except the entity / relation scatter.
//
// Bounds: the serial backward keeps two C-channel maps (one padded to a 401-float channel stride), the image and
// one weight bank in shared memory — acre_tr_serial_smem(C) <= 227 KB, i.e. C <= 46, the inference trunk's bound;
// the parallel way takes C <= ACRE_TR_PAR_MAX.
#pragma once
#include "kge_acre.cuh"
#include "kge_conve_train.cuh"

namespace kge {

constexpr int ACRE_TR_PAR_MAX = 1024;    // parallel way: largest in_channels (the gate rows Q*C stay one GEMM)
constexpr int ACRE_TR_INSTRIDE = ACRE_PIX + 1;   // channel stride of the weight-gradient input map (bank spread)

struct AcreTrain {
  const float* ent; const float* rel;
  const int64_t* e; const int64_t* r;
  int C; int dil[3]; bool par; bool has_bias;
  long long Q, B;                // rows, rows per group
  const float* bn0_w; const float* bn0_b;
  const float* conv_w[3]; const float* conv_b[3];
  const float* bn1_w; const float* bn1_b;
  const float* noise0;           // [Q, 400] or NULL
  const float* noise1;           // [Q, C] or NULL
  // workspace (forward writes, backward reads; the backward's scratch follows)
  float* img;                    // [Q, 400]   raw stacked rows
  float* y;                      // [Q, C*400] bn1's input
  float* feat;                   // [Q, C*400] feat; in the backward d feat -> g1 -> dy
  float* a1; float* a2;          // serial: [Q, C*400] conv1 and conv2 outputs
  float* gate;                   // parallel: [Q*C, 1600] gate rows; in the backward d gate
  float* st0; float* st1;        // [G, 2], [G, C, 2]
  float* part0; float* part1;    // [Q, 2], [Q, C, 2]
  float* red1;                   // [G, C, 2]
  float* dimg;                   // [Q, 400]   d (bn0 output)
  float* pw[3]; float* pb[3];    // per-query d conv_l.weight [Q, C*Cin*9], d conv_l.bias [Q, C]
};

struct AcreTrainLayout {
  long long img, y, feat, a1, a2, gate, partial, hpre, st0, st1, st2, part0, part1, red0, red1, dh, dimg;
  long long pw[3], pb[3], total;
};

inline int acre_tr_cin(int l, int C, bool par) { return (l == 0 || par) ? 1 : C; }

// float offsets of the workspace regions, each 64-float aligned (16-byte loads of the GEMM operands)
inline AcreTrainLayout acre_train_layout(long long Q, long long B, int C, bool par) {
  const long long Fw = (long long)C * ACRE_PIX, S = conve_fc_slices(Fw), G = Q / B;
  AcreTrainLayout L{};
  long long o = 0;
  auto take = [&o](long long n) { const long long at = o; o += (n + 63) / 64 * 64; return at; };
  L.img = take(Q * ACRE_PIX); L.y = take(Q * Fw); L.feat = take(Q * Fw);
  L.a1 = take(par ? 0 : Q * Fw); L.a2 = take(par ? 0 : Q * Fw); L.gate = take(par ? Q * C * ACRE_GATE : 0);
  L.partial = take(S * Q * ACRE_K); L.hpre = take(Q * ACRE_K);
  L.st0 = take(G * 2); L.st1 = take(G * C * 2); L.st2 = take(G * ACRE_K * 2);
  L.part0 = take(Q * 2); L.part1 = take(Q * C * 2); L.red0 = take(G * 2); L.red1 = take(G * C * 2);
  L.dh = take(Q * ACRE_K); L.dimg = take(Q * ACRE_PIX);
  for (int l = 0; l < 3; ++l) {
    L.pw[l] = take(Q * C * acre_tr_cin(l, C, par) * 9);
    L.pb[l] = take(Q * C);
  }
  L.total = o;
  return L;
}

// Serial kernels' shared memory, in floats: the image v [400], two map slots of C channels (401 floats each: one
// holds maps at stride 400, the other the weight-gradient input at stride 401), one weight bank [9][C][Cpad] and a
// bias row [Cpad].  4 * (400 + 802 C + 9 C ceil8(C) + ceil8(C)) bytes: C <= 46 within 227 KB.
struct AcreTrainSmem { long long img, a, b, w, bias, total; };

__host__ __device__ inline AcreTrainSmem acre_tr_serial_smem(int C) {
  const long long Cp = acre_cpad(C), slot = ((long long)C * ACRE_TR_INSTRIDE + 3) / 4 * 4;
  AcreTrainSmem S;
  S.img = 0;
  S.a = ACRE_PIX;
  S.b = S.a + slot;
  S.w = S.b + slot;                              // 16-byte aligned: the bank is read as float4
  S.bias = S.w + 9 * C * Cp;
  S.total = S.bias + Cp;
  return S;
}

// Gate kernels' shared memory, in floats: the image v [400], the three banks [3][C][9], then (forward only) the three
// bias rows [3][C]
__host__ __device__ inline long long acre_tr_gate_smem(int C) { return ACRE_PIX + 30ll * C; }
__host__ __device__ inline long long acre_tr_gate_bwd_smem(int C) { return ACRE_PIX + 27ll * C; }

// the fields the reused ConvE kernels read (gather, bn0 backward, bn2 forward / backward), AcrE's
inline ConveTrain acre_tr_view(const AcreTrain& a, const float* bn2_w, const float* bn2_b, const float* noise2,
                               float* hpre, float* st2, float* red0) {
  ConveTrain v{};
  v.ent = a.ent; v.rel = a.rel; v.e = a.e; v.r = a.r;
  v.k = ACRE_K; v.h2 = 10; v.h1 = 20; v.Q = a.Q; v.B = a.B;
  v.bn0_w = a.bn0_w; v.bn0_b = a.bn0_b; v.bn2_w = bn2_w; v.bn2_b = bn2_b; v.noise2 = noise2;
  v.img = a.img; v.hpre = hpre; v.st0 = a.st0; v.st2 = st2; v.part0 = a.part0; v.red0 = red0; v.dimg = a.dimg;
  return v;
}

// v = bn0(img) * noise0 of query q into v[400]; no barrier inside
KGE_DEV void acre_tr_stage_v(const AcreTrain& a, long long q, float* v, int nthreads) {
  const long long g = q / a.B;
  const float mean = a.st0[g * 2], invstd = a.st0[g * 2 + 1], w = __ldg(a.bn0_w), b = __ldg(a.bn0_b);
  for (int i = threadIdx.x; i < ACRE_PIX; i += nthreads) {
    float x = conve_bn_apply(a.img[q * ACRE_PIX + i], mean, invstd, w, b);
    if (a.noise0) x = fmul(x, __ldg(a.noise0 + q * ACRE_PIX + i));
    v[i] = x;
  }
}

KGE_DEV void acre_tr_store_map(const float* m, float* out, int C, int tid) {
  for (int i = tid; i < C * ACRE_PIX; i += ACRE_THREADS) out[i] = m[i];
}

__global__ void __launch_bounds__(ACRE_THREADS) acre_tr_serial_kernel(const AcreTrain a) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else   // host emulation: __shared__ is a function-local static there, so it needs a fixed size
  __shared__ float4 smem_f4[ACRE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const long long q = blockIdx.x;
  const int tid = threadIdx.x, C = a.C, Cp = acre_cpad(C);
  const long long Fw = (long long)C * ACRE_PIX;
  const AcreTrainSmem S = acre_tr_serial_smem(C);
  float* v = sm + S.img;
  float* ma = sm + S.a;
  float* mb = sm + S.b;
  float* w = sm + S.w;
  float* bias = sm + S.bias;
  acre_tr_stage_v(a, q, v, ACRE_THREADS);
  acre_stage_bank(a.conv_w[0], a.conv_b[0], 1, C, Cp, w, bias, tid, ACRE_THREADS);
  __syncthreads();
  acre_conv_layer<false>(v, 1, C, Cp, a.dil[0], a.has_bias, w, bias, ma, nullptr, nullptr, nullptr, nullptr, tid);
  __syncthreads();
  acre_tr_store_map(ma, a.a1 + q * Fw, C, tid);
  acre_stage_bank(a.conv_w[1], a.conv_b[1], C, C, Cp, w, bias, tid, ACRE_THREADS);
  __syncthreads();
  acre_conv_layer<false>(ma, C, C, Cp, a.dil[1], a.has_bias, w, bias, mb, nullptr, nullptr, nullptr, nullptr, tid);
  __syncthreads();
  acre_tr_store_map(mb, a.a2 + q * Fw, C, tid);
  acre_stage_bank(a.conv_w[2], a.conv_b[2], C, C, Cp, w, bias, tid, ACRE_THREADS);
  __syncthreads();
  acre_conv_layer<false>(mb, C, C, Cp, a.dil[2], a.has_bias, w, bias, ma, nullptr, nullptr, nullptr, nullptr, tid);
  __syncthreads();
  float* y = a.y + q * Fw;
  for (int i = tid; i < C * ACRE_PIX; i += ACRE_THREADS) y[i] = fadd(ma[i], v[i % ACRE_PIX]);
}

// parallel way: v, then the C gate rows [v ; conv1(v)[c] ; conv2(v)[c] ; conv3(v)[c]] of the query (kge_acre.cuh's
// acre_gate_input_kernel on the batch-statistics image).  The three banks [3][C][9] into w, the bias rows [3][C] into
// bias unless it is NULL (the backward needs no biases)
KGE_DEV void acre_tr_stage_gate_banks(const AcreTrain& a, float* w, float* bias) {
  const int C = a.C;
  for (int i = threadIdx.x; i < 27 * C; i += blockDim.x) {
    const int l = i / (9 * C), rest = i - l * 9 * C;
    w[i] = __ldg(a.conv_w[l] + rest);
  }
  if (bias)
    for (int i = threadIdx.x; i < 3 * C; i += blockDim.x) {
      const int l = i / C;
      bias[i] = a.has_bias ? __ldg(a.conv_b[l] + (i - l * C)) : 0.f;
    }
}

__global__ void __launch_bounds__(ACRE_GATE_THREADS) acre_tr_gate_kernel(const AcreTrain a) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[ACRE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const long long q = blockIdx.x;
  const int C = a.C;
  float* v = sm;
  float* w = sm + ACRE_PIX;          // [3][C][9]
  float* bias = w + 27 * C;          // [3][C]
  acre_tr_stage_v(a, q, v, ACRE_GATE_THREADS);
  acre_tr_stage_gate_banks(a, w, bias);
  __syncthreads();
  float* out = a.gate + q * C * ACRE_GATE;
  for (int o = threadIdx.x; o < C * ACRE_GATE; o += ACRE_GATE_THREADS) {
    const int c = o / ACRE_GATE, rem = o - c * ACRE_GATE, seg = rem / ACRE_PIX, px = rem - seg * ACRE_PIX;
    float y;
    if (seg == 0) {
      y = v[px];
    } else {
      const int l = seg - 1, d = a.dil[l], i = px / ACRE_SIDE, j = px - i * ACRE_SIDE;
      const float* wc = w + (l * C + c) * 9;
      float acc = 0.f;
      for (int u = 0; u < 3; ++u) {
        const int ii = i + (u - 1) * d;
        if (ii < 0 || ii >= ACRE_SIDE) continue;
        for (int t = 0; t < 3; ++t) {
          const int jj = j + (t - 1) * d;
          if (jj < 0 || jj >= ACRE_SIDE) continue;
          acc = ffma(wc[u * 3 + t], v[ii * ACRE_SIDE + jj], acc);
        }
      }
      y = a.has_bias ? fadd(acc, bias[l * C + c]) : acc;
    }
    out[o] = y;
  }
}

// one CTA (256 threads) per query, one warp per channel: bn1's per-query partials of y
__global__ void __launch_bounds__(CONVE_TR_THREADS) acre_tr_bn1_part_kernel(const AcreTrain a) {
  const long long q = blockIdx.x;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C;
  for (int c = warp; c < C; c += CONVE_TR_THREADS / 32) {
    const float* yc = a.y + (q * C + c) * ACRE_PIX;
    float s = 0.f;
    for (int p = lane; p < ACRE_PIX; p += 32) s = fadd(s, yc[p]);
    s = conve_warp_sum(s);
    const float m = __fdiv_rn(s, (float)ACRE_PIX);
    float m2 = 0.f;
    for (int p = lane; p < ACRE_PIX; p += 32) {
      const float d = fsub(yc[p], m);
      m2 = ffma(d, d, m2);
    }
    m2 = conve_warp_sum(m2);
    if (lane == 0) { a.part1[(q * C + c) * 2] = s; a.part1[(q * C + c) * 2 + 1] = m2; }
  }
}

__global__ void __launch_bounds__(256) acre_tr_feat_kernel(const AcreTrain a) {
  const long long Fw = (long long)a.C * ACRE_PIX, i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.Q * Fw) return;
  const long long q = i / Fw;
  const int c = (int)((i - q * Fw) / ACRE_PIX);
  const float* st = a.st1 + ((q / a.B) * a.C + c) * 2;
  float v = fmaxf(conve_bn_apply(__ldg(a.y + i), st[0], st[1], __ldg(a.bn1_w + c), __ldg(a.bn1_b + c)), 0.f);
  if (a.noise1) v = fmul(v, __ldg(a.noise1 + q * a.C + c));
  a.feat[i] = v;
}

// ---- backward ------------------------------------------------------------------------------------------------

// one CTA per query: feat's buffer holds d feat -> g1 = d (bn1 output) in place, the relu mask recomputed from y;
// per-channel (sum g1, sum g1 xhat1) partials
__global__ void __launch_bounds__(CONVE_TR_THREADS) acre_tr_bn1_bwd_part_kernel(const AcreTrain a) {
  const long long q = blockIdx.x, g = q / a.B;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, C = a.C;
  for (int c = warp; c < C; c += CONVE_TR_THREADS / 32) {
    const float* st = a.st1 + (g * C + c) * 2;
    const float mean = st[0], invstd = st[1], w = __ldg(a.bn1_w + c), b = __ldg(a.bn1_b + c);
    const float nz = a.noise1 ? __ldg(a.noise1 + q * C + c) : 1.0f;
    float* dc = a.feat + (q * C + c) * ACRE_PIX;
    const float* yc = a.y + (q * C + c) * ACRE_PIX;
    float sg = 0.f, sgx = 0.f;
    for (int p = lane; p < ACRE_PIX; p += 32) {
      const float xhat = fmul(fsub(__ldg(yc + p), mean), invstd);
      const float g1 = ffma(xhat, w, b) > 0.f ? (a.noise1 ? fmul(dc[p], nz) : dc[p]) : 0.f;
      dc[p] = g1;
      sg = fadd(sg, g1);
      sgx = ffma(g1, xhat, sgx);
    }
    sg = conve_warp_sum(sg);
    sgx = conve_warp_sum(sgx);
    if (lane == 0) { a.part1[(q * C + c) * 2] = sg; a.part1[(q * C + c) * 2 + 1] = sgx; }
  }
}

// dy = bn1 backward of g1, in place (elementwise)
__global__ void __launch_bounds__(256) acre_tr_bn1_bwd_kernel(const AcreTrain a) {
  const long long Fw = (long long)a.C * ACRE_PIX, i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= a.Q * Fw) return;
  const long long q = i / Fw, g = q / a.B;
  const int c = (int)((i - q * Fw) / ACRE_PIX);
  const float* st = a.st1 + (g * a.C + c) * 2;
  const float* rd = a.red1 + (g * a.C + c) * 2;
  const float inv_n1 = __fdiv_rn(1.0f, fmul((float)a.B, (float)ACRE_PIX));
  const float xhat = fmul(fsub(__ldg(a.y + i), st[0]), st[1]);
  a.feat[i] = conve_bn_bwd(a.feat[i], xhat, rd[0], rd[1], inv_n1, __ldg(a.bn1_w + c), st[1]);
}

// Per-query weight gradient of one dilated 3x3 layer (Cin -> C): pw[(co*Cin + ci)*9 + t] = sum over the pixels p
// whose tap t lands inside the image of dz[co][p] * in[ci][p + shift_t]; pb[co] = sum_p dz[co][p].  dz: maps at
// stride 400; in: maps at stride `is`.  Warp item (tap, 8 output channels, 32 input channels): lane = 8 * phase + h
// holds input channels 4h..4h+3 of the block over the columns j = j0 + phase + 4m; the 4 phases are added by
// shuffles at the end.  Only whole warps take part (warp < ACRE_THREADS / 32).
KGE_DEV void acre_tr_wgrad(const float* dz, const float* in, int is, int Cin, int C, int d, float* pw, float* pb,
                           int tid) {
  const int lane = tid & 31, warp = tid >> 5, h = lane & 7, phase = lane >> 3;
  const int G = (C + ACRE_CB - 1) / ACRE_CB, H = (Cin + 31) / 32, items = 9 * G * H;
  if (warp < ACRE_THREADS / 32) {
    for (int it = warp; it < items; it += ACRE_THREADS / 32) {
      const int t = it / (G * H), rest = it - t * G * H, g = rest / H, hb = rest - g * H;
      const int du = (t / 3 - 1) * d, dv = (t % 3 - 1) * d;
      const int i0 = max(0, -du), i1 = min(ACRE_SIDE, ACRE_SIDE - du);
      const int j0 = max(0, -dv), j1 = min(ACRE_SIDE, ACRE_SIDE - dv);
      const int ci0 = hb * 32 + h * 4;
      int cz[ACRE_CB], cx[4];
#pragma unroll
      for (int b = 0; b < ACRE_CB; ++b) cz[b] = min(g * ACRE_CB + b, C - 1) * ACRE_PIX;
#pragma unroll
      for (int m = 0; m < 4; ++m) cx[m] = min(ci0 + m, Cin - 1) * is + du * ACRE_SIDE + dv;
      float acc[ACRE_CB][4];
#pragma unroll
      for (int b = 0; b < ACRE_CB; ++b)
#pragma unroll
        for (int m = 0; m < 4; ++m) acc[b][m] = 0.f;
      for (int i = i0; i < i1; ++i) {
        for (int j = j0 + phase; j < j1; j += 4) {
          const int p = i * ACRE_SIDE + j;
          float x[4];
#pragma unroll
          for (int m = 0; m < 4; ++m) x[m] = in[cx[m] + p];
#pragma unroll
          for (int b = 0; b < ACRE_CB; ++b) {
            const float z = dz[cz[b] + p];
#pragma unroll
            for (int m = 0; m < 4; ++m) acc[b][m] = ffma(z, x[m], acc[b][m]);
          }
        }
      }
#pragma unroll
      for (int b = 0; b < ACRE_CB; ++b)
#pragma unroll
        for (int m = 0; m < 4; ++m) {
          float s = acc[b][m];
          s = fadd(s, __shfl_xor_sync(0xffffffffu, s, 8));
          s = fadd(s, __shfl_xor_sync(0xffffffffu, s, 16));
          const int co = g * ACRE_CB + b, ci = ci0 + m;
          if (phase == 0 && co < C && ci < Cin) pw[((long long)co * Cin + ci) * 9 + t] = s;
        }
    }
  }
  if (pb)
    for (int co = tid; co < C; co += ACRE_THREADS) {
      float s = 0.f;
      for (int p = 0; p < ACRE_PIX; ++p) s = fadd(s, dz[co * ACRE_PIX + p]);
      pb[co] = s;
    }
}

// the transposed bank of layer W [C][Cin][3][3] for the data gradient, a conv C -> Cin with the taps flipped:
// wt[(t*C + co)*Cpi + ci] = W[co][ci][8 - t] (zero for ci >= Cin), Cpi = ceil8(Cin)
KGE_DEV void acre_tr_stage_bank_t(const float* __restrict__ cw, int Cin, int C, float* wt, int tid) {
  const int Cpi = acre_cpad(Cin), n = 9 * C * Cpi;
  for (int i = tid; i < n; i += ACRE_THREADS) {
    const int ci = i % Cpi, rest = i / Cpi, co = rest % C, t = rest / C;
    wt[i] = ci < Cin ? __ldg(cw + ((long long)co * Cin + ci) * 9 + (8 - t)) : 0.f;
  }
}

// the input map of a layer's weight gradient into shared memory at channel stride ACRE_TR_INSTRIDE
KGE_DEV void acre_tr_load_in(const float* src, float* dst, int Cin, int tid) {
  for (int i = tid; i < Cin * ACRE_PIX; i += ACRE_THREADS) {
    const int c = i / ACRE_PIX;
    dst[i + c] = src[i];
  }
}

// serial way, one CTA per query: layers 3, 2, 1 in turn — the per-query weight / bias gradients from dz_l and the
// layer's input, then d (input) = the transposed conv of dz_l, which is dz_{l-1}; d v = d a0 + sum_c dy[c]
__global__ void __launch_bounds__(ACRE_THREADS) acre_tr_serial_bwd_kernel(const AcreTrain a) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[ACRE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const long long q = blockIdx.x;
  const int tid = threadIdx.x, C = a.C;
  const long long Fw = (long long)C * ACRE_PIX;
  const AcreTrainSmem S = acre_tr_serial_smem(C);
  float* v = sm + S.img;
  float* dz = sm + S.a;        // this layer's output gradient, stride 400
  float* xin = sm + S.b;       // this layer's input, stride 401; then its gradient, stride 400
  float* w = sm + S.w;
  const float* dy = a.feat + q * Fw;
  for (int i = tid; i < C * ACRE_PIX; i += ACRE_THREADS) dz[i] = dy[i];
  acre_tr_load_in(a.a2 + q * Fw, xin, C, tid);
  acre_tr_stage_v(a, q, v, ACRE_THREADS);
  __syncthreads();
  float res = 0.f;   // the residual's gradient sum_c dy[c][tid] (thread tid owns pixel tid)
  for (int c = 0; c < C; ++c) res = fadd(res, dz[c * ACRE_PIX + tid]);
  for (int l = 2; l >= 0; --l) {
    const int Cin = l == 0 ? 1 : C;
    const float* in = l == 0 ? v : xin;
    const int is = l == 0 ? ACRE_PIX : ACRE_TR_INSTRIDE;
    acre_tr_stage_bank_t(a.conv_w[l], Cin, C, w, tid);
    acre_tr_wgrad(dz, in, is, Cin, C, a.dil[l], a.pw[l] + q * C * Cin * 9, a.has_bias ? a.pb[l] + q * C : nullptr,
                  tid);
    __syncthreads();   // the bank is staged; every read of xin as the layer's input is done
    acre_conv_layer<false>(dz, C, Cin, acre_cpad(Cin), a.dil[l], false, w, nullptr, xin, nullptr, nullptr, nullptr,
                           nullptr, tid);
    __syncthreads();   // d (input) complete in xin; dz is free
    if (l == 0) break;
    float* tmp = dz; dz = xin; xin = tmp;
    if (l == 2) acre_tr_load_in(a.a1 + q * Fw, xin, C, tid);
    __syncthreads();
  }
  // xin holds d a0 (one channel, stride 400)
  float dv = fadd(xin[tid], res);
  if (a.noise0) dv = fmul(dv, __ldg(a.noise0 + q * ACRE_PIX + tid));
  a.dimg[q * ACRE_PIX + tid] = dv;
}

// parallel way, one CTA per query: d gate [Q*C, 1600] holds (d v, dz1, dz2, dz3) per channel.  Per-query gradients
// of the three 1 -> C convs (one chain over the pixels per element), then d v = sum_c d gate[c][0] + the transposed
// convs (sum over c ascending, then layer, then tap), * noise0 -> dimg
__global__ void __launch_bounds__(ACRE_GATE_THREADS) acre_tr_gate_bwd_kernel(const AcreTrain a) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[ACRE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const long long q = blockIdx.x;
  const int C = a.C;
  float* v = sm;
  float* w = sm + ACRE_PIX;
  acre_tr_stage_v(a, q, v, ACRE_GATE_THREADS);
  acre_tr_stage_gate_banks(a, w, nullptr);
  __syncthreads();
  const float* dg = a.gate + q * C * ACRE_GATE;
  const int nb = a.has_bias ? 3 * C : 0;
  for (int it = threadIdx.x; it < 27 * C + nb; it += ACRE_GATE_THREADS) {
    if (it < 27 * C) {
      const int l = it / (9 * C), rest = it - l * 9 * C, c = rest / 9, t = rest - c * 9, d = a.dil[l];
      const int du = (t / 3 - 1) * d, dv = (t % 3 - 1) * d;
      const int i0 = max(0, -du), i1 = min(ACRE_SIDE, ACRE_SIDE - du);
      const int j0 = max(0, -dv), j1 = min(ACRE_SIDE, ACRE_SIDE - dv);
      const float* dz = dg + (long long)c * ACRE_GATE + (l + 1) * ACRE_PIX;
      float s = 0.f;
      for (int i = i0; i < i1; ++i)
        for (int j = j0; j < j1; ++j) {
          const int p = i * ACRE_SIDE + j;
          s = ffma(dz[p], v[p + du * ACRE_SIDE + dv], s);
        }
      a.pw[l][q * C * 9 + rest] = s;
    } else {
      const int b = it - 27 * C, l = b / C, c = b - l * C;
      const float* dz = dg + (long long)c * ACRE_GATE + (l + 1) * ACRE_PIX;
      float s = 0.f;
      for (int p = 0; p < ACRE_PIX; ++p) s = fadd(s, dz[p]);
      a.pb[l][q * C + c] = s;
    }
  }
  for (int px = threadIdx.x; px < ACRE_PIX; px += ACRE_GATE_THREADS) {
    const int I = px / ACRE_SIDE, J = px - I * ACRE_SIDE;
    float acc = 0.f;
    for (int c = 0; c < C; ++c) acc = fadd(acc, dg[(long long)c * ACRE_GATE + px]);
    for (int l = 0; l < 3; ++l) {
      const int d = a.dil[l];
      for (int c = 0; c < C; ++c) {
        const float* dz = dg + (long long)c * ACRE_GATE + (l + 1) * ACRE_PIX;
        const float* wc = w + (l * C + c) * 9;
        for (int u = 0; u < 3; ++u) {
          const int i = I - (u - 1) * d;
          if (i < 0 || i >= ACRE_SIDE) continue;
          for (int t = 0; t < 3; ++t) {
            const int j = J - (t - 1) * d;
            if (j < 0 || j >= ACRE_SIDE) continue;
            acc = ffma(wc[u * 3 + t], dz[i * ACRE_SIDE + j], acc);
          }
        }
      }
    }
    if (a.noise0) acc = fmul(acc, __ldg(a.noise0 + q * ACRE_PIX + px));
    a.dimg[q * ACRE_PIX + px] = acc;
  }
}

// one CTA (256 threads) per query: bn0's backward partials (sum g, sum g xhat0) of dimg (CTA sums)
__global__ void __launch_bounds__(CONVE_TR_THREADS) acre_tr_bn0_part_kernel(const AcreTrain a) {
  __shared__ float sh[CONVE_TR_THREADS / 32];
  const long long q = blockIdx.x, g = q / a.B;
  const float mean0 = a.st0[g * 2], invstd0 = a.st0[g * 2 + 1];
  float s0 = 0.f, s1 = 0.f;
  for (int px = threadIdx.x; px < ACRE_PIX; px += CONVE_TR_THREADS) {
    const float d = a.dimg[q * ACRE_PIX + px];
    s0 = fadd(s0, d);
    s1 = ffma(d, fmul(fsub(a.img[q * ACRE_PIX + px], mean0), invstd0), s1);
  }
  s0 = conve_block_sum(s0, sh);
  s1 = conve_block_sum(s1, sh);
  if (threadIdx.x == 0) { a.part0[q * 2] = s0; a.part0[q * 2 + 1] = s1; }
}

}  // namespace kge
