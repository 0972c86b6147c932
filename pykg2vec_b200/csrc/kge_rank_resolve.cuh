// kge_rank_resolve.cuh — level 2 of the 1-vs-all rank: exact re-evaluation of listed (query, candidate)
// pairs with the canonical fp32 group function.  Shared by the filter pass of the gather and fp32 paths
// (resolve_pairs_kernel, kge_rank.cu) and by the tensor-core path's resolve-and-commit kernel
// (kge_rank_tiled.cu).
#pragma once
#include "kge_models.cuh"
#include "kge_rank.cuh"

namespace kge {

constexpr int kResolveThreads = 256;
constexpr int kResolveGroups = kResolveThreads / 8;

// One direction's pairs to resolve.  With a band list (tensor-core path) ctrl is the list's control block:
// [0] length, [1] overflow, [2] the resolve-and-commit kernel's done counter.
struct ResolveArgs {
  const int64_t *qh, *qr, *qt;
  const float* thr;                  // [Q] thresholds: the target's own score
  const unsigned long long* list;    // band list (q << 32 | local candidate row), or nullptr
  unsigned* ctrl;
  unsigned cap;                      // band-list capacity
  int32_t* tc_counts;                // [Q] counts of the tensor-core levels
  RankFilter F;
  int64_t Q, row_lo, row_hi;
  int32_t* counts;                   // [Q][4]
  int col, scratch_floats;
};

// launch parameters of the group-function kernels (kge_rank.cu)
struct GroupArgs { ModelParams P; int vec, sf; size_t smem; };
GroupArgs group_args(const RankCall& C);
ResolveArgs resolve_args(const RankCall& C, int dir);

// One 8-lane group per item, grid-stride over the kernel's groups:
//   items [0, total)            : band-list pairs: tc_counts[q] += 1 when the candidate really outranks the target
//   items [total, total + nnz)  : the filter entries: the filtered column -= 1 when the entry outranks the
//                                 target.  Entries equal to the target or outside the row shard are skipped.
template <int MODEL, int VEC, int GROUPING>
KGE_DEV void resolve_items(const ModelParams& P, const ResolveArgs& A, int64_t total, float* scratch) {
  const RankFilter& F = A.F;
  const int lane = threadIdx.x & 7;
  // the true entry count lives in device memory (ptr[Q]); the host may pass a capacity
  // (upper bound) as nnz so that the launch shape can stay fixed inside a CUDA graph
  const int64_t nnz_true = (F.ptr && F.idx && F.nnz > 0) ? min(F.nnz, __ldg(F.ptr + A.Q)) : 0;
  const int64_t items = total + nnz_true;
  for (int64_t k = (int64_t)blockIdx.x * kResolveGroups + (threadIdx.x >> 3); k < items;
       k += (int64_t)gridDim.x * kResolveGroups) {
    int64_t q, e;
    bool skip = false;
    const bool band = k < total;
    if (band) {
      const unsigned long long pr = A.list[k];
      if (pr == ~0ull) continue;   // unused slot of a warp's reserved block (kge_rank_tc.cu); group-uniform
      q = (int64_t)(pr >> 32);
      e = (int64_t)(pr & 0xffffffffull);
    } else {
      const int64_t kk = k - total;
      int64_t lo = 0, hi = A.Q;  // largest q with ptr[q] <= kk
      while (hi - lo > 1) {
        const int64_t mid = (lo + hi) >> 1;
        if (__ldg(F.ptr + mid) <= kk) lo = mid; else hi = mid;
      }
      q = lo;
      const int64_t ge = __ldg(F.idx + kk);
      skip = (ge == __ldg(F.tgt + q)) || ge < A.row_lo || ge >= A.row_hi;
      e = skip ? 0 : ge - A.row_lo;
    }
    TripleRows R;
    if (GROUPING == KGE_GROUP_TAIL)
      resolve_rows<MODEL>(R, P, P.qtab, P.tab, P.qtab, __ldg(A.qh + q), __ldg(A.qr + q), e);
    else
      resolve_rows<MODEL>(R, P, P.tab, P.qtab, P.qtab, e, __ldg(A.qr + q), __ldg(A.qt + q));
    prefetch_triple_rows(R, P.d, P.dr, lane);
    const float s = score_group<MODEL, VEC, GROUPING>(R, P, lane, scratch);
    if (lane == 0 && !skip && s < __ldg(A.thr + q)) {
      if (band) atomicAdd(A.tc_counts + q, 1);
      else atomicSub(A.counts + q * 4 + A.col + 1, 1);
    }
  }
}

}  // namespace kge
