// kge_acre.cuh — AcrE's trunk in inference mode (AcrE.forward, pykg2vec/models/projection.py:706-734 with
// self.training == False: dropouts are identities, bn0 / bn1 / bn2 use their running statistics):
//     img[20][20] = bn0([ent[e] ; rel[r]])            the two 200-wide rows read as 10 x 20 each, stacked
//     conv_l = 3x3 conv, stride 1, padding = dilation = atrous_l (zero padding: the output stays 20 x 20)
//     serial:   y = conv3(conv2(conv1(img))) + img    1 -> C -> C -> C channels, img broadcast over the C
//                                                     channels (acre_serial_feature_kernel below)
//     parallel: g[c] = [img ; conv1(img)[c] ; conv2(img)[c] ; conv3(img)[c]]   1600 values per channel, each
//                                                     conv 1 -> C (acre_gate_input_kernel below)
//               y[c] = W_gate_e(g[c])                 the tiled GEMM of kge_proj.cuh, bias in the epilogue
//     feat = relu(bn1(y)) flattened channel-major     (fused into the serial kernel; acre_bn1_relu_kernel for
//                                                     the parallel way)
//     x = relu(bn2(feat . fc.weight^T + fc.bias))     ConvE's sliced Linear GEMM + hyper_fc_combine_kernel
// Canonical arithmetic (restated by tests/oracle_acre/kge_oracle_acre.c, bit for bit):
//     BatchNorm(v) = fma(v, a, c) with a = w / sqrt(var + eps), c = b - mean * a (bn_fold);
//     conv output (co, i, j) = one sequential fma chain from 0 in TAP-MAJOR order: tap (u, v) row-major, and
//     within a tap the input channels ci = 0..Cin-1, of w[co][ci][u][v] * in[ci][i + (u-1)d][j + (v-1)d].
//     Taps that fall in the zero padding are SKIPPED (no fma at all), then + conv bias as a separate add when
//     acre_bias is set.  (Tap-major, because whether a tap is inside the image depends on the pixel and the tap
//     only: the channel loop inside a tap runs without a per-channel test.);
//     serial: the residual is a separate add, conv3 + img, then the bn1 fold of the channel, then max(., 0);
//     parallel: W_gate_e = one fma chain over the 1600 gate inputs in order from 0, then + W_gate_e.bias (the
//     tiled GEMM's rule), then the bn1 fold of channel c, then max(., 0);
//     feature index c * 400 + i * 20 + j;
//     Linear and combine = HypER's (kge_hyper.cuh): one fma chain per slice of CONVE_FC_SLICE features, slice
//     sums added in ascending order, then + fc.bias, then the bn2 fold, then relu.
#pragma once
#include "kge_hyper.cuh"

namespace kge {

constexpr int ACRE_SIDE = 20;                  // the image is 20 x 20 (two 10 x 20 halves)
constexpr int ACRE_PIX = ACRE_SIDE * ACRE_SIDE;
constexpr int ACRE_K = 200;                    // hidden_size: the only size whose rows make that image
constexpr int ACRE_GATE = 4 * ACRE_PIX;        // W_gate_e input width, 1600 (hard-coded in the reference)
constexpr int ACRE_THREADS = 400;              // serial kernel
constexpr int ACRE_CB = 8;                     // output channels per thread (the weight bank is padded to 8)
constexpr int ACRE_PB = 4;                     // pixels per thread: rows i, i+5, i+10, i+15 of one column
constexpr int ACRE_ITEMS_PER_GROUP = ACRE_PIX / ACRE_PB;   // 100 thread items per group of 8 channels
constexpr int ACRE_GATE_THREADS = 256;         // parallel gate-input kernel
constexpr int ACRE_SMEM_MAX = 227 * 1024;      // bytes: the per-block opt-in maximum of sm_90

struct AcreFeat {
  const float* ent; const float* rel;          // [N, 200], [2R, 200]
  const int64_t* e; const int64_t* r;
  int C; int dil[3];                           // in_channels, first / second / third atrous
  const float* bn0_w; const float* bn0_b; const float* bn0_mean; const float* bn0_var; float bn0_eps;
  const float* conv_w[3];                      // serial [C,1,3,3], [C,C,3,3], [C,C,3,3]; parallel 3 x [C,1,3,3]
  const float* conv_b[3];                      // [C] each, or all null (acre_bias = False)
  const float* bn1_w; const float* bn1_b; const float* bn1_mean; const float* bn1_var; float bn1_eps;
  float* out;                                  // serial: features [Q, C*400]; parallel: gate input [Q*C, 1600]
};

__host__ __device__ inline int acre_cpad(int C) { return (C + ACRE_CB - 1) / ACRE_CB * ACRE_CB; }

// Serial kernel's shared memory, in floats: the bn0 image [400], two C x 400 maps (conv1 and conv2 outputs),
// one weight bank [9][Cin][Cpad] (tap-major, zero columns co >= C; restaged for each layer), the layer's
// conv bias [Cpad] and the bn1 folds a1 / c1 [Cpad].  Total 400 + 800 C + 9 C Cpad + 3 Cpad floats, Cpad =
// ceil8(C): 141 KB at C = 32.  It fits the 227 KB opt-in while
//     4 * (400 + 800*C + 9*C*ceil8(C) + 3*ceil8(C)) <= 232448,  i.e.  C <= 46.
struct AcreSmem { long long img, a, b, w, bias, a1, c1, total; };

__host__ __device__ inline AcreSmem acre_serial_smem(int C) {
  const long long Cp = acre_cpad(C);
  AcreSmem S;
  S.img = 0;
  S.a = ACRE_PIX;
  S.b = S.a + (long long)C * ACRE_PIX;
  S.w = S.b + (long long)C * ACRE_PIX;         // 16-byte aligned: 400 + 800 C is a multiple of 4
  S.bias = S.w + 9 * C * Cp;
  S.a1 = S.bias + Cp;
  S.c1 = S.a1 + Cp;
  S.total = S.c1 + Cp;
  return S;
}

// Gate-input kernel's shared memory, in floats: the bn0 image [400], the three banks [3][C][9], the three
// bias rows [3][C].
__host__ __device__ inline long long acre_gate_smem(int C) { return ACRE_PIX + 30ll * C; }

// bn0 of the stacked [ent ; rel] rows into img[400]
KGE_DEV void acre_stage_image(const AcreFeat& p, int q, float* img, int tid, int nthreads) {
  float a0, c0;
  bn_fold(__ldg(p.bn0_w), __ldg(p.bn0_b), __ldg(p.bn0_mean), __ldg(p.bn0_var), p.bn0_eps, a0, c0);
  const float* er = p.ent + __ldg(p.e + q) * (long long)ACRE_K;
  const float* rr = p.rel + __ldg(p.r + q) * (long long)ACRE_K;
  for (int i = tid; i < ACRE_PIX; i += nthreads)
    img[i] = ffma(i < ACRE_K ? __ldg(er + i) : __ldg(rr + (i - ACRE_K)), a0, c0);
}

// conv weights [C][Cin][3][3] -> w[(t*Cin + ci)*Cp + co] (tap-major, zero for co >= C); bias [Cp] (0 if none)
KGE_DEV void acre_stage_bank(const float* __restrict__ cw, const float* __restrict__ cb, int Cin, int C, int Cp,
                             float* w, float* bias, int tid, int nthreads) {
  const int n = 9 * Cin * Cp;
  for (int i = tid; i < n; i += nthreads) {
    const int co = i % Cp, rest = i / Cp, ci = rest % Cin, t = rest / Cin;
    w[i] = co < C ? __ldg(cw + ((long long)co * Cin + ci) * 9 + t) : 0.f;
  }
  for (int i = tid; i < Cp; i += nthreads) bias[i] = (cb && i < C) ? __ldg(cb + i) : 0.f;
}

// One dilated 3x3 conv layer, Cin -> C channels, over maps of 400 floats per channel in shared memory.  Thread
// item (g, s): channels 8g..8g+7 at the pixels s, s+100, s+200, s+300 (rows i0 + 5m of column j).  Per tap
// inside the image and per input channel: four image reads (consecutive pixels across the warp), two float4
// reads of the bank (one address per group across the warp) and 32 fma.  FINAL: + res, bn1 fold, relu and
// the channel-major store to global memory; otherwise the raw conv (+ bias) into `out` in shared memory.
template <bool FINAL>
KGE_DEV void acre_conv_layer(const float* in, int Cin, int C, int Cp, int d, bool has_bias, const float* w,
                             const float* bias, float* out, const float* res, const float* a1, const float* c1,
                             float* gout, int tid) {
  const int items = Cp / ACRE_CB * ACRE_ITEMS_PER_GROUP;
  for (int it = tid; it < items; it += ACRE_THREADS) {
    const int g = it / ACRE_ITEMS_PER_GROUP, s = it - g * ACRE_ITEMS_PER_GROUP;
    const int i0 = s / ACRE_SIDE, j = s - i0 * ACRE_SIDE;
    float acc[ACRE_PB][ACRE_CB];
#pragma unroll
    for (int m = 0; m < ACRE_PB; ++m)
#pragma unroll
      for (int b = 0; b < ACRE_CB; ++b) acc[m][b] = 0.f;
    for (int u = 0; u < 3; ++u) {
      for (int v = 0; v < 3; ++v) {
        const int jj = j + (v - 1) * d;
        if (jj < 0 || jj >= ACRE_SIDE) continue;          // the whole column of taps is padding
        bool ok[ACRE_PB];
        int off[ACRE_PB];
#pragma unroll
        for (int m = 0; m < ACRE_PB; ++m) {
          const int ii = i0 + 5 * m + (u - 1) * d;
          ok[m] = ii >= 0 && ii < ACRE_SIDE;
          off[m] = ok[m] ? ii * ACRE_SIDE + jj : 0;
        }
        const float* wp = w + (u * 3 + v) * Cin * Cp + g * ACRE_CB;
        const float* ip = in;
#pragma unroll 4
        for (int ci = 0; ci < Cin; ++ci, wp += Cp, ip += ACRE_PIX) {
          const float4 w0 = *reinterpret_cast<const float4*>(wp);
          const float4 w1 = *reinterpret_cast<const float4*>(wp + 4);
#pragma unroll
          for (int m = 0; m < ACRE_PB; ++m) {
            if (!ok[m]) continue;
            const float x = ip[off[m]];
            acc[m][0] = ffma(w0.x, x, acc[m][0]); acc[m][1] = ffma(w0.y, x, acc[m][1]);
            acc[m][2] = ffma(w0.z, x, acc[m][2]); acc[m][3] = ffma(w0.w, x, acc[m][3]);
            acc[m][4] = ffma(w1.x, x, acc[m][4]); acc[m][5] = ffma(w1.y, x, acc[m][5]);
            acc[m][6] = ffma(w1.z, x, acc[m][6]); acc[m][7] = ffma(w1.w, x, acc[m][7]);
          }
        }
      }
    }
#pragma unroll
    for (int m = 0; m < ACRE_PB; ++m) {
      const int px = s + m * ACRE_ITEMS_PER_GROUP;
#pragma unroll
      for (int b = 0; b < ACRE_CB; ++b) {
        const int co = g * ACRE_CB + b;
        if (co >= C) continue;
        float y = acc[m][b];
        if (has_bias) y = fadd(y, bias[co]);
        if (FINAL)
          gout[co * ACRE_PIX + px] = fmaxf(ffma(fadd(y, res[px]), a1[co], c1[co]), 0.f);
        else
          out[co * ACRE_PIX + px] = y;
      }
    }
  }
}

// serial way, one CTA per query: gather + bn0, conv1 -> conv2 -> conv3 with each layer's bank staged in shared
// memory, + residual, bn1 fold, relu, channel-major store of the C*400 features
__global__ void __launch_bounds__(ACRE_THREADS) acre_serial_feature_kernel(const AcreFeat p) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else   // host emulation (tests/emu): __shared__ is a function-local static there, so it needs a fixed size
  __shared__ float4 smem_f4[ACRE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const int q = blockIdx.x, tid = threadIdx.x, C = p.C, Cp = acre_cpad(C);
  const AcreSmem S = acre_serial_smem(C);
  float* img = sm + S.img;
  float* ma = sm + S.a;
  float* mb = sm + S.b;
  float* w = sm + S.w;
  float* bias = sm + S.bias;
  float* a1 = sm + S.a1;
  float* c1 = sm + S.c1;
  const bool has_bias = p.conv_b[0] != nullptr;
  acre_stage_image(p, q, img, tid, ACRE_THREADS);
  acre_stage_bank(p.conv_w[0], p.conv_b[0], 1, C, Cp, w, bias, tid, ACRE_THREADS);
  for (int c = tid; c < Cp; c += ACRE_THREADS) {
    if (c < C)
      bn_fold(__ldg(p.bn1_w + c), __ldg(p.bn1_b + c), __ldg(p.bn1_mean + c), __ldg(p.bn1_var + c), p.bn1_eps,
              a1[c], c1[c]);
    else
      a1[c] = c1[c] = 0.f;
  }
  __syncthreads();
  acre_conv_layer<false>(img, 1, C, Cp, p.dil[0], has_bias, w, bias, ma, nullptr, nullptr, nullptr, nullptr, tid);
  __syncthreads();
  acre_stage_bank(p.conv_w[1], p.conv_b[1], C, C, Cp, w, bias, tid, ACRE_THREADS);
  __syncthreads();
  acre_conv_layer<false>(ma, C, C, Cp, p.dil[1], has_bias, w, bias, mb, nullptr, nullptr, nullptr, nullptr, tid);
  __syncthreads();
  acre_stage_bank(p.conv_w[2], p.conv_b[2], C, C, Cp, w, bias, tid, ACRE_THREADS);
  __syncthreads();
  acre_conv_layer<true>(mb, C, C, Cp, p.dil[2], has_bias, w, bias, nullptr, img, a1, c1,
                        p.out + (long long)q * C * ACRE_PIX, tid);
}

// parallel way, one CTA per query: gather + bn0, then the C gate-input rows [img ; conv1[c] ; conv2[c] ;
// conv3[c]] of the query, each conv 1 -> C with its own dilation (9 taps, padding skipped, + bias)
__global__ void __launch_bounds__(ACRE_GATE_THREADS) acre_gate_input_kernel(const AcreFeat p) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[ACRE_SMEM_MAX / 16];
#endif
  float* sm = reinterpret_cast<float*>(smem_f4);
  const int q = blockIdx.x, tid = threadIdx.x, C = p.C;
  float* img = sm;
  float* w = sm + ACRE_PIX;          // [3][C][9]
  float* bias = w + 27 * C;          // [3][C]
  const bool has_bias = p.conv_b[0] != nullptr;
  acre_stage_image(p, q, img, tid, ACRE_GATE_THREADS);
  for (int i = tid; i < 27 * C; i += ACRE_GATE_THREADS) {
    const int l = i / (9 * C), rest = i - l * 9 * C;
    w[i] = __ldg(p.conv_w[l] + rest);
  }
  for (int i = tid; i < 3 * C; i += ACRE_GATE_THREADS) {
    const int l = i / C;
    bias[i] = has_bias ? __ldg(p.conv_b[l] + (i - l * C)) : 0.f;
  }
  __syncthreads();
  float* out = p.out + (long long)q * C * ACRE_GATE;
  for (int o = tid; o < C * ACRE_GATE; o += ACRE_GATE_THREADS) {
    const int c = o / ACRE_GATE, rem = o - c * ACRE_GATE, seg = rem / ACRE_PIX, px = rem - seg * ACRE_PIX;
    float y;
    if (seg == 0) {
      y = img[px];
    } else {
      const int l = seg - 1, d = p.dil[l], i = px / ACRE_SIDE, j = px - i * ACRE_SIDE;
      const float* wc = w + (l * C + c) * 9;
      float acc = 0.f;
      for (int u = 0; u < 3; ++u) {
        const int ii = i + (u - 1) * d;
        if (ii < 0 || ii >= ACRE_SIDE) continue;
        for (int v = 0; v < 3; ++v) {
          const int jj = j + (v - 1) * d;
          if (jj < 0 || jj >= ACRE_SIDE) continue;
          acc = ffma(wc[u * 3 + v], img[ii * ACRE_SIDE + jj], acc);
        }
      }
      y = has_bias ? fadd(acc, bias[l * C + c]) : acc;
    }
    out[o] = y;
  }
}

// y[i] = relu(bn1_c(y[i])) in place over the W_gate_e output [Q*C, 400], channel c = row % C
__global__ void __launch_bounds__(256)
acre_bn1_relu_kernel(float* __restrict__ y, long long n, int C, const float* __restrict__ bn1_w,
                     const float* __restrict__ bn1_b, const float* __restrict__ bn1_mean,
                     const float* __restrict__ bn1_var, float bn1_eps) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= n) return;
  const int c = (int)((i / ACRE_PIX) % C);
  float a1, c1;
  bn_fold(__ldg(bn1_w + c), __ldg(bn1_b + c), __ldg(bn1_mean + c), __ldg(bn1_var + c), bn1_eps, a1, c1);
  y[i] = fmaxf(ffma(y[i], a1, c1), 0.f);
}

// ---- launch plans: plain C++ shared by the C-ABI launcher (kge_proj.cu) and the CPU emulation test ---------
// Workspace, in floats: the gate input [Q*C, 1600] (parallel way only, else empty), the features [Q, C*400]
// (the parallel way's W_gate_e output, made features in place by acre_bn1_relu_kernel), the Linear layer's
// slice partials [slices, Q, 200].  Every region starts 16-byte aligned.
struct AcreLayout { long long gate, feat, partial, total; };

inline long long acre_feat_width(int C) { return (long long)C * ACRE_PIX; }

inline AcreLayout acre_layout(long long Q, int C, bool parallel) {
  const long long Fw = acre_feat_width(C);
  AcreLayout L;
  L.gate = 0;
  L.feat = parallel ? Q * C * ACRE_GATE : 0;
  L.partial = L.feat + Q * Fw;
  L.total = L.partial + (long long)conve_fc_slices(Fw) * Q * ACRE_K;
  return L;
}

// y[Q*C, 400] = gate[Q*C, 1600] . W_gate_e[400, 1600]^T + bias   (one chain over the 1600 inputs, no activation)
inline ProjLaunch acre_plan_gate(const float* gate, const float* wg, const float* bg, long long rows, float* y,
                                 int tile) {
  ProjLaunch L = proj_plan_fwd(gate, wg, bg, rows, ACRE_PIX, ACRE_GATE, y, tile);
  L.g.act = ACT_NONE;
  return L;
}

}  // namespace kge
