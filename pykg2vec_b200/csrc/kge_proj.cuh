// kge_proj.cuh — kernels + launch plans of the tail every projection model of the reference shares (SURVEY.md §8 a11 / f4):
//     preds = sigmoid(x . E^T + b)                 ConvE.inner_forward  projection.py:100-102
//     (TuckER :335-336, InteractE :444-447, HypER :607-609, AcrE :735-738; ProjE g() :248-256)
//     Criterion.multi_class_bce                    criterion.py:41-50
//     predict_tail_rank / predict_head_rank        projection.py:119-125  (+ evaluator.py:70-123)
// as one register-tiled fp32 GEMM kernel with three epilogues:
//     EPI_STORE    store act(acc + bias), act = sigmoid | relu      -> forward(); ConvE's Linear layer
//     EPI_COUNT    count sigmoid(acc + bias) > target pred per row  -> rank counts, no [Q,N] matrix
//     EPI_ATOMIC   accumulate acc into C (split-K)                  -> grad_x, grad_ent
// Canonical arithmetic (DESIGN.md §3 rule 8): an output element is ONE sequential fma chain over
// the contraction index starting from 0 — exactly the order this tiling accumulates in (k-chunks
// ascending, kk ascending inside a chunk; zero padding is an exact identity) — then one add of
// the bias and the canonical sigmoid.  oracle/kge_oracle.c (proj_pred) restates it; the two agree
// bit for bit, so the counts of EPI_COUNT equal counting over the forward() matrix.
#pragma once
#include "kge_common.cuh"

namespace kge {

constexpr int PBM = 64, PBN = 64;   // the 64x64 CTA tile (gradient and Linear-layer launches; smallest forward tile)
constexpr int PBK = 16, PTHREADS = 256;
enum { EPI_STORE = 0, EPI_ATOMIC = 1, EPI_COUNT = 2 };
enum { ACT_SIGMOID = 0, ACT_RELU = 1, ACT_NONE = 2 };

// C(m,n) = sum_k A(m,k) * B(n,k) with A(m,k) = A[m*sAm + k*sAk], B(n,k) = B[n*sBn + k*sBk].
struct ProjGemm {
  const float* A; long long sAm, sAk;
  const float* Ap;      // optional, indexed like A: A(m,k) is multiplied by p(1-p) (d sigmoid)
  const float* B; long long sBn, sBk;
  int M, N, K, klen;    // klen = contraction range per blockIdx.z (multiple of PBK)
  int avec, bvec;       // 16-byte loads along k are legal for A / B
  float* C; long long ldc;
  long long zstride;    // STORE: slice blockIdx.z writes to C + blockIdx.z * zstride (partial products)
  const float* bias;    // [N] or null (STORE, COUNT)
  int act;              // STORE: ACT_SIGMOID, ACT_RELU or ACT_NONE
  const float* thr;     // COUNT: [M] prediction of the target
  int* counts;          // COUNT: counts[m*4 + coff] and [m*4 + coff + 1] += #better
  int coff;
};

// Staging of a [ROWS x PBK] operand tile, k-major in shared memory (S[kk][row]), in two halves
// so that the global loads of chunk c+1 are in flight while chunk c is multiplied: fetch() reads
// this thread's ROWS/16 elements into registers, place() writes them to shared memory.  Rows / k
// beyond the operand read as 0 (an exact identity for the fma chain).
template <int ROWS>
struct ProjRegs { float v[ROWS / 16]; };

template <int ROWS>
KGE_DEV void proj_fetch_tile(ProjRegs<ROWS>& R, const float* __restrict__ P, const float* __restrict__ Pp,
                             long long sr, long long sk, bool usevec, int r0, int nrows, int k0,
                             int kend, int tid) {
  static_assert(ROWS % 64 == 0, "whole 16-byte loads per thread");
  constexpr int PER = ROWS / 16;   // elements per thread (ROWS * PBK / PTHREADS)
  if (usevec) {  // sk == 1, rows 16-byte aligned: 16-byte load f -> (row f/4, 4 consecutive k)
#pragma unroll
    for (int u = 0; u < PER / 4; ++u) {
      const int f = tid + u * PTHREADS;
      const int rr = f >> 2, kq = (f & 3) * 4;
      const int gr = r0 + rr, gk = k0 + kq;
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
      if (gr < nrows && gk < kend) {
        const float* src = P + (long long)gr * sr + gk;
        if (gk + 3 < kend) {
          v = __ldg(reinterpret_cast<const float4*>(src));
        } else {
          v.x = __ldg(src);
          if (gk + 1 < kend) v.y = __ldg(src + 1);
          if (gk + 2 < kend) v.z = __ldg(src + 2);
        }
      }
      R.v[4 * u + 0] = v.x; R.v[4 * u + 1] = v.y; R.v[4 * u + 2] = v.z; R.v[4 * u + 3] = v.w;
    }
    return;
  }
  const bool kcontig = (sk == 1);
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    const int i = tid + u * PTHREADS;
    int rr, kk;
    if (kcontig) { kk = i % PBK; rr = i / PBK; } else { rr = i % ROWS; kk = i / ROWS; }
    const int gr = r0 + rr, gk = k0 + kk;
    float v = 0.f;
    if (gr < nrows && gk < kend) {
      const long long off = (long long)gr * sr + (long long)gk * sk;
      v = __ldg(P + off);
      if (Pp) { const float p = __ldg(Pp + off); v = fmul(v, fmul(p, fsub(1.0f, p))); }
    }
    R.v[u] = v;
  }
}

template <int ROWS>
KGE_DEV void proj_place_tile(float (*S)[ROWS + 4], const ProjRegs<ROWS>& R, long long sk, bool usevec, int tid) {
  constexpr int PER = ROWS / 16;
  if (usevec) {
#pragma unroll
    for (int u = 0; u < PER / 4; ++u) {
      const int f = tid + u * PTHREADS;
      const int rr = f >> 2, kq = (f & 3) * 4;
#pragma unroll
      for (int e = 0; e < 4; ++e) S[kq + e][rr] = R.v[4 * u + e];
    }
    return;
  }
  const bool kcontig = (sk == 1);
#pragma unroll
  for (int u = 0; u < PER; ++u) {
    const int i = tid + u * PTHREADS;
    int rr, kk;
    if (kcontig) { kk = i % PBK; rr = i / PBK; } else { rr = i % ROWS; kk = i / ROWS; }
    S[kk][rr] = R.v[u];
  }
}

// Thread (ty, tx) of the 16x16 thread grid owns TM x TN outputs of the (16*TM) x (16*TN) CTA tile,
// in groups of 4 consecutive rows / columns 64 apart: row(i) = (i/4)*64 + ty*4 + i%4, likewise
// col(j) with tx — so every shared-memory operand read is one conflict-free 16-byte load per group
// and a half-warp covers 64 consecutive output columns.
template <int EPI, int TM, int TN>
__global__ void __launch_bounds__(PTHREADS) proj_gemm_kernel(const ProjGemm g) {
  constexpr int BM = 16 * TM, BN = 16 * TN;
  __shared__ __align__(16) float As[PBK][BM + 4];
  __shared__ __align__(16) float Bs[PBK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
  const int kbeg = blockIdx.z * g.klen;
  const int kend = min(g.K, kbeg + g.klen);
  const bool avec = g.avec && !g.Ap, bvec = g.bvec != 0;
  float acc[TM][TN];
#pragma unroll
  for (int i = 0; i < TM; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  ProjRegs<BM> ra;
  ProjRegs<BN> rb;
  if (kbeg < kend) {
    proj_fetch_tile<BM>(ra, g.A, g.Ap, g.sAm, g.sAk, avec, m0, g.M, kbeg, kend, tid);
    proj_fetch_tile<BN>(rb, g.B, nullptr, g.sBn, g.sBk, bvec, n0, g.N, kbeg, kend, tid);
  }
  for (int k0 = kbeg; k0 < kend; k0 += PBK) {
    proj_place_tile<BM>(As, ra, g.sAk, avec, tid);
    proj_place_tile<BN>(Bs, rb, g.sBk, bvec, tid);
    __syncthreads();
    if (k0 + PBK < kend) {  // next chunk's loads overlap this chunk's multiply
      proj_fetch_tile<BM>(ra, g.A, g.Ap, g.sAm, g.sAk, avec, m0, g.M, k0 + PBK, kend, tid);
      proj_fetch_tile<BN>(rb, g.B, nullptr, g.sBn, g.sBk, bvec, n0, g.N, k0 + PBK, kend, tid);
    }
#pragma unroll
    for (int kk = 0; kk < PBK; ++kk) {
      float av[TM], bv[TN];
#pragma unroll
      for (int gi = 0; gi < TM / 4; ++gi) {
        const float4 a4 = *reinterpret_cast<const float4*>(&As[kk][gi * 64 + ty * 4]);
        av[4 * gi + 0] = a4.x; av[4 * gi + 1] = a4.y; av[4 * gi + 2] = a4.z; av[4 * gi + 3] = a4.w;
      }
#pragma unroll
      for (int gj = 0; gj < TN / 4; ++gj) {
        const float4 b4 = *reinterpret_cast<const float4*>(&Bs[kk][gj * 64 + tx * 4]);
        bv[4 * gj + 0] = b4.x; bv[4 * gj + 1] = b4.y; bv[4 * gj + 2] = b4.z; bv[4 * gj + 3] = b4.w;
      }
#pragma unroll
      for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = ffma(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < TM; ++i) {
    const int gm = m0 + (i / 4) * 64 + ty * 4 + (i % 4);
    if (EPI == EPI_COUNT) {
      int c = 0;
      if (gm < g.M) {
        const float th = __ldg(g.thr + gm);
#pragma unroll
        for (int j = 0; j < TN; ++j) {
          const int gn = n0 + (j / 4) * 64 + tx * 4 + (j % 4);
          if (gn < g.N) {
            float l = acc[i][j];
            if (g.bias) l = fadd(l, __ldg(g.bias + gn));
            c += (sigmoid_canon(l) > th) ? 1 : 0;
          }
        }
      }
      // the 16 threads sharing this output row are the 16 lanes of one half-warp
      c += __shfl_xor_sync(0xffffffffu, c, 8);
      c += __shfl_xor_sync(0xffffffffu, c, 4);
      c += __shfl_xor_sync(0xffffffffu, c, 2);
      c += __shfl_xor_sync(0xffffffffu, c, 1);
      if (tx == 0 && gm < g.M && c) {
        atomicAdd(g.counts + (long long)gm * 4 + g.coff, c);
        atomicAdd(g.counts + (long long)gm * 4 + g.coff + 1, c);
      }
    } else {
      if (gm >= g.M) continue;
#pragma unroll
      for (int j = 0; j < TN; ++j) {
        const int gn = n0 + (j / 4) * 64 + tx * 4 + (j % 4);
        if (gn >= g.N) continue;
        float* dst = g.C + (long long)blockIdx.z * g.zstride + (long long)gm * g.ldc + gn;
        if (EPI == EPI_STORE) {
          float l = acc[i][j];
          if (g.bias) l = fadd(l, __ldg(g.bias + gn));
          *dst = (g.act == ACT_SIGMOID) ? sigmoid_canon(l) : (g.act == ACT_RELU ? fmaxf(l, 0.f) : l);
        } else {
          atomicAdd(dst, acc[i][j]);
        }
      }
    }
  }
}

// prediction of each query's target entity, by the same fma chain as the GEMM
__global__ void __launch_bounds__(128)
proj_target_kernel(const float* __restrict__ x, const float* __restrict__ ent,
                   const float* __restrict__ bias, const int64_t* __restrict__ tgt, int Q, int k,
                   float* __restrict__ thr) {
  const int q = blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= Q) return;
  const int64_t e = __ldg(tgt + q);
  const float* xr = x + (long long)q * k;
  const float* er = ent + e * (long long)k;
  float acc = 0.f;
  for (int j = 0; j < k; ++j) acc = ffma(__ldg(xr + j), __ldg(er + j), acc);
  if (bias) acc = fadd(acc, __ldg(bias + e));
  thr[q] = sigmoid_canon(acc);
}

// filtered rank = raw - #{e in filter row, e != target : pred(e) > pred(target)}; one CTA per query
__global__ void __launch_bounds__(128)
proj_filter_kernel(const float* __restrict__ x, const float* __restrict__ ent,
                   const float* __restrict__ bias, const int64_t* __restrict__ tgt,
                   const int64_t* __restrict__ ptr, const int64_t* __restrict__ idx, int k,
                   const float* __restrict__ thr, int* __restrict__ counts, int coff) {
  __shared__ int total;
  const int q = blockIdx.x;
  if (threadIdx.x == 0) total = 0;
  __syncthreads();
  const int64_t beg = __ldg(ptr + q), end = __ldg(ptr + q + 1), t = __ldg(tgt + q);
  const float th = __ldg(thr + q);
  const float* xr = x + (long long)q * k;
  int c = 0;
  for (int64_t p = beg + threadIdx.x; p < end; p += blockDim.x) {
    const int64_t e = __ldg(idx + p);
    if (e == t) continue;
    const float* er = ent + e * (long long)k;
    float acc = 0.f;
    for (int j = 0; j < k; ++j) acc = ffma(__ldg(xr + j), __ldg(er + j), acc);
    if (bias) acc = fadd(acc, __ldg(bias + e));
    c += (sigmoid_canon(acc) > th) ? 1 : 0;
  }
  if (c) atomicAdd(&total, c);
  __syncthreads();
  if (threadIdx.x == 0 && total) atomicSub(counts + (long long)q * 4 + coff + 1, total);
}

// one direction of Criterion.multi_class_bce: value + d loss / d preds
__global__ void __launch_bounds__(256)
proj_bce_kernel(const float* __restrict__ preds, const float* __restrict__ labels, long long n,
                float label_scale, float label_shift, float gs, float inv_count,
                float* __restrict__ loss, float* __restrict__ gpreds) {
  __shared__ float red[8];
  float acc = 0.f;
  for (long long i = (long long)blockIdx.x * 256 + threadIdx.x; i < n; i += (long long)gridDim.x * 256) {
    const float z = __ldg(preds + i);
    const float y = fadd(fmul(__ldg(labels + i), label_scale), label_shift);
    const float sp = fadd(fmaxf(-z, 0.f), log_canon(fadd(1.0f, exp_canon(-fabsf(z)))));
    acc += ffma(fsub(1.0f, y), z, sp);
    if (gpreds) gpreds[i] = fmul(fsub(sigmoid_canon(z), y), gs);
  }
#pragma unroll
  for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) s += red[w];
    atomicAdd(loss, s * inv_count);
  }
}

// grad_bias[n] += sum_b grad_preds[b,n] * p (1 - p)
__global__ void __launch_bounds__(256)
proj_colsum_kernel(const float* __restrict__ gp, const float* __restrict__ preds, int B, long long N,
                   float* __restrict__ gb) {
  const long long n = (long long)blockIdx.x * 256 + threadIdx.x;
  if (n >= N) return;
  float acc = 0.f;
  for (int b = 0; b < B; ++b) {
    const long long off = (long long)b * N + n;
    const float p = __ldg(preds + off);
    acc = ffma(__ldg(gp + off), fmul(p, fsub(1.0f, p)), acc);
  }
  gb[n] += acc;
}

// Dense multi-class label rows from CSR rows of known positives: labels[b, idx[p]] = 1 for p in
// [ptr[row], ptr[row+1]), row = rows[b] (or b when rows is null); the buffer is zero-filled before.
// What process_function_multiclass builds on the host per batch (generator.py:160-236, neg_rate 0).
__global__ void __launch_bounds__(128)
proj_labels_kernel(const int64_t* __restrict__ rows, const int64_t* __restrict__ ptr,
                   const int64_t* __restrict__ idx, long long N, float* __restrict__ labels) {
  const long long b = blockIdx.x;
  const int64_t row = rows ? __ldg(rows + b) : b;
  const int64_t beg = __ldg(ptr + row), end = __ldg(ptr + row + 1);
  for (int64_t p = beg + threadIdx.x; p < end; p += blockDim.x) labels[b * N + __ldg(idx + p)] = 1.0f;
}

// ---- launch plans: plain C++ (shared by the C-ABI launchers in kge_proj.cu and by the CPU
// emulation test tests/emu/, which runs these kernels thread by thread on the host) ------------
// CTA tile variants of proj_gemm_kernel: rows x columns (thread tile = rows/16 x columns/16)
enum { PROJ_TILE_64x64 = 0, PROJ_TILE_64x128 = 1, PROJ_TILE_128x128 = 2 };
inline int proj_tile_rows(int tile) { return tile == PROJ_TILE_128x128 ? 128 : 64; }
inline int proj_tile_cols(int tile) { return tile == PROJ_TILE_64x64 ? 64 : 128; }
// Large tiles halve the shared-memory operand traffic per fma (a 16-byte read feeds 32 fma instead
// of 16) but need enough CTAs to fill every SM: the largest tile that still gives two CTAs per SM.
inline int proj_pick_tile(long long M, long long N, int sms) {
  if (((M + 127) / 128) * ((N + 127) / 128) >= 2ll * sms) return PROJ_TILE_128x128;
  if (((M + 63) / 64) * ((N + 127) / 128) >= (long long)sms) return PROJ_TILE_64x128;
  return PROJ_TILE_64x64;
}

struct ProjLaunch { ProjGemm g; unsigned gx, gy, gz; int tile; };

inline int proj_vec_ok(const float* p, long long row_stride, long long k_stride) {
  return k_stride == 1 && (row_stride % 4 == 0) && (((uintptr_t)p & 15) == 0);
}
inline unsigned proj_tiles(long long n, int tile) { return (unsigned)((n + tile - 1) / tile); }

// preds[B,N] = sigmoid(x[B,k] . ent[N,k]^T + bias)   — also the frame of the counting launch
inline ProjLaunch proj_plan_fwd(const float* x, const float* ent, const float* bias, long long B,
                                long long N, int k, float* preds, int tile = PROJ_TILE_64x64) {
  ProjLaunch L{};
  L.tile = tile;
  ProjGemm& g = L.g;
  g.A = x; g.sAm = k; g.sAk = 1; g.Ap = nullptr;
  g.B = ent; g.sBn = k; g.sBk = 1;
  g.M = (int)B; g.N = (int)N; g.K = k; g.klen = (int)proj_tiles(k, PBK) * PBK;
  g.avec = proj_vec_ok(x, k, 1); g.bvec = proj_vec_ok(ent, k, 1);
  g.C = preds; g.ldc = N; g.bias = bias; g.act = ACT_SIGMOID;
  L.gx = proj_tiles(N, proj_tile_cols(tile)); L.gy = proj_tiles(B, proj_tile_rows(tile)); L.gz = 1;
  return L;
}

inline ProjLaunch proj_plan_count(const float* x, const float* ent, const float* bias, long long Q,
                                  long long N, int k, const float* thr, int* counts, int direction,
                                  int tile = PROJ_TILE_64x64) {
  ProjLaunch L = proj_plan_fwd(x, ent, bias, Q, N, k, nullptr, tile);
  L.g.thr = thr; L.g.counts = counts; L.g.coff = 2 * direction;
  return L;
}

// grad_x[B,k] += g[B,N] . ent[N,k]: contraction over the entities, split over `target_ctas` CTAs
inline ProjLaunch proj_plan_grad_x(const float* grad_preds, const float* preds, const float* ent,
                                   long long B, long long N, int k, float* grad_x, int target_ctas) {
  ProjLaunch L{};
  ProjGemm& g = L.g;
  g.A = grad_preds; g.sAm = N; g.sAk = 1; g.Ap = preds;
  g.B = ent; g.sBn = 1; g.sBk = k;
  g.M = (int)B; g.N = k; g.K = (int)N;
  const long long tiles = (long long)proj_tiles(B, PBM) * proj_tiles(k, PBN);
  const long long chunks = proj_tiles(N, PBK);
  long long splits = (target_ctas + tiles - 1) / tiles;
  if (splits > chunks) splits = chunks;
  if (splits < 1) splits = 1;
  const long long per = (chunks + splits - 1) / splits;
  g.klen = (int)(per * PBK);
  g.avec = 0; g.bvec = 0;
  g.C = grad_x; g.ldc = k;
  L.gx = proj_tiles(k, PBN); L.gy = proj_tiles(B, PBM); L.gz = (unsigned)((chunks + per - 1) / per);
  return L;
}

// grad_ent[N,k] += g^T[N,B] . x[B,k]
inline ProjLaunch proj_plan_grad_ent(const float* grad_preds, const float* preds, const float* x,
                                     long long B, long long N, int k, float* grad_ent) {
  ProjLaunch L{};
  ProjGemm& g = L.g;
  g.A = grad_preds; g.sAm = 1; g.sAk = N; g.Ap = preds;
  g.B = x; g.sBn = 1; g.sBk = k;
  g.M = (int)N; g.N = k; g.K = (int)B; g.klen = (int)proj_tiles(B, PBK) * PBK;
  g.avec = 0; g.bvec = 0;
  g.C = grad_ent; g.ldc = k;
  L.gx = proj_tiles(k, PBN); L.gy = proj_tiles(N, PBM); L.gz = 1;
  return L;
}

// Criterion.multi_class_bce scalars, computed in double as the reference's Python floats are
inline float proj_bce_grad_factor(float grad_scale, long long B, long long N) {
  return (float)((double)grad_scale / ((double)B * (double)N));
}
inline float proj_bce_inv_count(long long B, long long N) { return (float)(1.0 / ((double)B * (double)N)); }
inline unsigned proj_bce_blocks(long long n, int sms) {
  long long blocks = (n + 255) / 256;
  const long long cap = 8ll * sms;
  return (unsigned)(blocks > cap ? cap : blocks);
}

}  // namespace kge
