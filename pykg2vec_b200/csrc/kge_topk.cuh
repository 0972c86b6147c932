// kge_topk.cuh — batched top-k link prediction: the k best tails, heads or relations of each query,
// raw or with a per-query filter of known positives left out.  Replaces the reference's one-query-at-a-time
// route (evaluator.py:249-287 test_*_rank, trainer.py:330-386 infer_*, projection.py:119-125
// predict_*_rank: one N-wide forward and a full sort per query, in descending forward score).
//
// Two stages per chunk of queries (launchers: kge_topk.cu):
//   producer   a [Qc, n] fp32 block of candidate scores in the workspace.  Kernel models:
//              topk_store_kernel below, score_group over (query, candidate) pairs exactly as the rank path's
//              gather sweep evaluates them; projection models: the tail GEMM's EPI_STORE launch (kge_proj.cuh).
//   select     topk_select_kernel, one CTA per row: the k smallest 64-bit keys (score key << 32 | id).
//
// Key order.  topk_score_key maps a score to a 32-bit key whose unsigned order is "better first": ascending
// score for the kernel models (lower is more plausible for every model), descending for the projection models'
// sigmoid.  -0 is folded onto +0, every NaN maps to 0xFFFFFFFF (after every number, +-inf included).  The id in
// the low word breaks ties towards the smaller id, so every row has one exact answer whatever the geometry.
//
// Selection (one CTA of 256 threads per row; thread t owns radix bin t):
//   1. the row's filter entries become a bitmap in shared memory (n bits); filtered candidates are not eligible;
//   2. four 8-bit-digit radix passes over the eligible score keys find T, the kk-th smallest score key
//      (kk = min(k, #eligible)), and how many of the keys equal to T belong to the answer (`need`);
//   3. one sweep collects every key below T and the `need` ties with the smallest ids.  When all ties are taken
//      the order of collection does not matter (step 4 sorts); when only some are, the ties are compacted in id
//      order by a block-wide exclusive scan per 256-candidate tile — no atomics decide which ties survive;
//   4. a bitonic sort of the <= 256 survivors in shared memory; ids and the scores (re-read from the row, so
//      -0 and NaN payloads keep their bits) are written best first, then id -1 / NaN up to k.
// The row stays in shared memory when it fits beside the bitmap (FB15k-237: 58 KB), else every pass streams it
// from the workspace (YAGO3-10's 123,182 entities: 493 KB per row).
#pragma once
#include "kge_models.cuh"

namespace kge {

constexpr int kTopkMaxK = 256;
constexpr int kTopkThreads = 256;                   // select: one thread per radix bin and per survivor slot
constexpr int kTopkGroups = kTopkThreads / 8;       // producer: 8-lane groups per CTA
constexpr int kTopkIters = 16;
constexpr int kTopkCandsPerCta = kTopkGroups * kTopkIters;
// Workspace bound: the launchers score at most this many bytes of candidates per chunk of queries (Qc rows of
// n candidates, Qc = max(1, floor(64 MiB / 4n)), at most 65535), so the workspace does not grow with Q.
constexpr long long kTopkChunkBytes = 64ll << 20;
constexpr long long kTopkMaxChunkRows = 65535;
// dynamic shared memory the select kernel may take (the 227 KB opt-in limit less its static arrays)
constexpr size_t kTopkSmemBudget = 227 * 1024 - 4 * 1024;
#ifndef __CUDACC__
// host emulation (tests/emu): __shared__ is a function-local static there, so the dynamic arrays get a fixed size
constexpr size_t kTopkEmuSmem = kTopkSmemBudget;
constexpr size_t kTopkEmuStoreSmem = 64 * 1024;
#endif

// ---- plain C++ plans, shared by the launchers and the host emulation ---------------------------------------
inline long long topk_chunk_rows(long long Q, long long n) {
  long long rows = kTopkChunkBytes / (4 * (n > 0 ? n : 1));
  if (rows < 1) rows = 1;
  if (rows > kTopkMaxChunkRows) rows = kTopkMaxChunkRows;
  return rows < Q ? rows : Q;
}
inline __host__ __device__ size_t topk_bitmap_bytes(long long n) { return (size_t)((n + 127) / 128) * 16; }
struct TopkSelectPlan { bool row_in_smem; size_t smem; };
// smem == 0: no plan (the bitmap alone does not fit; the launchers refuse such n)
inline TopkSelectPlan topk_select_plan(long long n) {
  const size_t bm = topk_bitmap_bytes(n);
  if (bm + (size_t)n * 4 <= kTopkSmemBudget) return {true, bm + (size_t)n * 4};
  if (bm <= kTopkSmemBudget) return {false, bm};
  return {false, 0};
}

// ---- score key ----------------------------------------------------------------------------------------------
KGE_DEV unsigned topk_score_key(float s, bool descending) {
  if (s != s) return 0xFFFFFFFFu;                     // NaN after every number
  if (descending) s = -s;
  unsigned u = __float_as_uint(s);
  if (u == 0x80000000u) u = 0u;                       // -0 == +0
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);  // order-preserving: negative floats reversed below positives
}

// ---- producer: candidate scores of the kernel models ---------------------------------------------------------
// TARGET 0: tails of (qh, qr) in TAIL grouping; 1: heads of (qr, qt) in HEAD grouping; 2: relations of (qh, qt)
// in TAIL grouping (kge_score_fwd's forward order).  One CTA = one query x kTopkCandsPerCta candidates; out is the
// [gridDim.y, n] block of this chunk's queries.
template <int MODEL, int VEC, int TARGET>
__global__ void __launch_bounds__(kTopkThreads)
topk_store_kernel(const ModelParams P, const int64_t* __restrict__ qh, const int64_t* __restrict__ qr,
                  const int64_t* __restrict__ qt, int64_t n, float* __restrict__ out, int scratch_floats) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[kTopkEmuStoreSmem / 16];
#endif
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const int64_t q = blockIdx.y;
  const int64_t h = TARGET == 1 ? 0 : __ldg(qh + q);
  const int64_t r = TARGET == 2 ? 0 : __ldg(qr + q);
  const int64_t t = TARGET == 0 ? 0 : __ldg(qt + q);
  const int64_t base = (int64_t)blockIdx.x * kTopkCandsPerCta;
  constexpr int GROUPING = TARGET == 1 ? KGE_GROUP_HEAD : KGE_GROUP_TAIL;
  for (int it = 0; it < kTopkIters; ++it) {
    const int64_t e = base + it * kTopkGroups + grp;
    const bool valid = e < n;
    const int64_t c = valid ? e : n - 1;   // idle groups shadow the last candidate (shuffles stay full-group)
    TripleRows R;
    if (TARGET == 0) resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, h, r, c);
    else if (TARGET == 1) resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, c, r, t);
    else resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, h, c, t);
    const float s = score_group<MODEL, VEC, GROUPING>(R, P, lane, scratch);
    if (valid && lane == 0) out[q * n + e] = s;
  }
}

// ---- selection ----------------------------------------------------------------------------------------------
struct TopkSelectArgs {
  const float* scores;      // [rows, n] this chunk's score block
  int64_t n;
  int k;
  bool descending;          // projection models: higher sigmoid first
  const int64_t* fptr;      // CSR filter rows of this chunk (ptr already offset to the chunk's first query) or NULL
  const int64_t* fidx;
  int64_t* ids;             // [rows, k] of this chunk
  float* out_scores;
};

// Inclusive prefix sum of v over the 256 threads of the block (xor butterfly inside each warp, then the warp
// totals through `wt`).  Returns the inclusive prefix; *total receives the block's sum.  Two barriers.
KGE_DEV int topk_block_scan(int v, int* wt, int* total) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int pre = v, tot = v;
#pragma unroll
  for (int off = 1; off < 32; off <<= 1) {
    const int o = __shfl_xor_sync(0xffffffffu, tot, off);
    if (lane & off) pre += o;
    tot += o;
  }
  if (lane == 0) wt[warp] = tot;
  __syncthreads();
  int before = 0, all = 0;
#pragma unroll
  for (int w = 0; w < kTopkThreads / 32; ++w) {
    const int x = wt[w];
    before += (w < warp) ? x : 0;
    all += x;
  }
  __syncthreads();   // wt may be rewritten by the next scan
  *total = all;
  return before + pre;
}

template <bool ROW_IN_SMEM>
__global__ void __launch_bounds__(kTopkThreads)
topk_select_kernel(const TopkSelectArgs A) {
#ifdef __CUDACC__
  extern __shared__ float4 smem_f4[];
#else
  __shared__ float4 smem_f4[kTopkEmuSmem / 16];
#endif
  __shared__ unsigned long long surv[kTopkMaxK];
  __shared__ int hist[256];
  __shared__ int wt[kTopkThreads / 32];
  __shared__ int s_digit, s_need, s_ties, s_cnt;
  const int tid = threadIdx.x;
  const int64_t q = blockIdx.x, n = A.n;
  unsigned* bm = reinterpret_cast<unsigned*>(smem_f4);
  const int64_t nwords = (n + 31) >> 5;
  const float* grow = A.scores + q * n;
  const float* row = grow;
  if (ROW_IN_SMEM) {
    float* srow = reinterpret_cast<float*>(smem_f4) + topk_bitmap_bytes(n) / 4;
    for (int64_t i = tid; i < n; i += kTopkThreads) srow[i] = __ldg(grow + i);
    row = srow;
  }
  for (int64_t w = tid; w < nwords; w += kTopkThreads) bm[w] = 0u;
  if (tid == 0) s_cnt = 0;
  __syncthreads();
  if (A.fptr) {
    const int64_t beg = __ldg(A.fptr + q), end = __ldg(A.fptr + q + 1);
    for (int64_t p = beg + tid; p < end; p += kTopkThreads) {
      const int64_t e = __ldg(A.fidx + p);
      if (e >= 0 && e < n) atomicOr(bm + (e >> 5), 1u << (e & 31));   // duplicates set the same bit
    }
  }
  __syncthreads();
  auto eligible = [&](int64_t i) { return ((bm[i >> 5] >> (i & 31)) & 1u) == 0u; };

  // 1-2: radix select of the kk-th smallest score key
  unsigned prefix = 0;
  int need = A.k, kk = 0;
  for (int pass = 0; pass < 4; ++pass) {
    const int shift = 24 - 8 * pass;
    hist[tid] = 0;
    __syncthreads();
    for (int64_t i = tid; i < n; i += kTopkThreads) {
      if (!eligible(i)) continue;
      const unsigned key = topk_score_key(row[i], A.descending);
      if (pass == 0 || (key >> (shift + 8)) == (prefix >> (shift + 8))) atomicAdd(hist + ((key >> shift) & 255u), 1);
    }
    __syncthreads();
    const int c = hist[tid];
    int total;
    const int incl = topk_block_scan(c, wt, &total);
    if (pass == 0) {
      kk = total < A.k ? total : A.k;   // fewer eligible candidates than k: all of them
      need = kk;
      if (kk == 0) break;               // (uniform) nothing eligible
    }
    if (incl - c < need && need <= incl) { s_digit = tid; s_need = need - (incl - c); s_ties = c; }
    __syncthreads();
    prefix |= (unsigned)s_digit << shift;
    need = s_need;
  }

  // 3: collect the keys below T and `need` ties, smallest ids first
  if (kk > 0) {
    const unsigned T = prefix;
    const int ties = s_ties;
    const bool ordered = ties > need;   // (uniform) only some of the ties survive
    const int c_less = kk - need;
    int tie_base = 0;
    for (int64_t i0 = 0; i0 < n; i0 += kTopkThreads) {
      const int64_t i = i0 + tid;
      const bool ok = i < n && eligible(i);
      const unsigned key = ok ? topk_score_key(row[i], A.descending) : 0xFFFFFFFFu;
      const bool lt = ok && key < T, tie = ok && key == T;
      const unsigned long long full = ((unsigned long long)key << 32) | (unsigned long long)(uint32_t)i;
      if (lt || (tie && !ordered)) surv[atomicAdd(&s_cnt, 1)] = full;
      if (ordered && tie_base < need) {   // (uniform)
        int tile_ties;
        const int pos = tie_base + topk_block_scan(tie ? 1 : 0, wt, &tile_ties) - 1;
        if (tie && pos < need) surv[c_less + pos] = full;
        tie_base += tile_ties;
      }
    }
  }
  // 4: bitonic sort of the survivors, padded with the largest key
  __syncthreads();
  if (tid >= kk) surv[tid] = ~0ull;
  for (int size = 2; size <= kTopkMaxK; size <<= 1) {
    for (int stride = size >> 1; stride > 0; stride >>= 1) {
      __syncthreads();
      const int p = tid ^ stride;
      if (p > tid) {
        const unsigned long long a = surv[tid], b = surv[p];
        const bool up = (tid & size) == 0;
        if ((a > b) == up) { surv[tid] = b; surv[p] = a; }
      }
    }
  }
  __syncthreads();
  if (tid < A.k) {
    int64_t id = -1;
    float s = __uint_as_float(0x7FC00000u);
    if (tid < kk) {
      id = (int64_t)(uint32_t)surv[tid];
      s = row[id];
    }
    A.ids[q * A.k + tid] = id;
    A.out_scores[q * A.k + tid] = s;
  }
}

}  // namespace kge
