// kge_rank.cuh — interface between the rank driver (kge_rank.cu), the fp32 tiled sweep
// (kge_rank_tiled.cu) and the tensor-core sweep (kge_rank_tc.cu): the workspace layout, the
// arguments of one rank call and the stages the driver runs for each direction.
#pragma once
#include "kge_common.cuh"

namespace kge {

// ---- model-level geometry ---------------------------------------------------------------------------
inline bool is_simple(int model) { return model == KGE_SIMPLE || model == KGE_SIMPLE_IGNR; }
// embedding width padded to whole 4-element chunks: row length of query vectors and candidate scratch
inline int rank_dp(const kge_model_t* m) { return ((m->dim + 3) / 4) * 4; }
// arrays per query vector and per candidate row of the tiled sweeps (KQ == KC): 2 for the two-term models
constexpr int rank_kq(int model) {
  return (model == KGE_ROTATE || model == KGE_COMPLEX || model == KGE_SIMPLE || model == KGE_SIMPLE_IGNR) ? 2 : 1;
}
bool tiled_supported(const kge_model_t* m);
bool tc_supported(const kge_model_t* m, int64_t nc);
// tensor-core operand kind: 0 dot, 1 squared distance (sum domain), 2 squared distance - margin
inline int tc_kind(const kge_model_t* m) { return (m->model == KGE_TRANSE) ? 1 : (m->model == KGE_ROTATE ? 2 : 0); }
// contraction length of the tensor-core operands: KQ arrays of dp (+ the three norm columns), padded to 16
inline int tc_kp(const kge_model_t* m) {
  const int K = rank_kq(m->model) * rank_dp(m) + (tc_kind(m) != 0 ? 3 : 0);
  return (K + 15) / 16 * 16;
}
// ambiguous-pair list slots per direction
inline unsigned tc_list_capacity(int64_t Q) {
  int64_t cap = 512 * Q;
  if (cap < 32768) cap = 32768;   // (every consumer warp reserves one block of 16 up front: <= one wave of CTAs x 8 x 16 slots)
  if (cap > (1 << 24)) cap = 1 << 24;
  return (unsigned)cap;
}

// ---- the workspace ----------------------------------------------------------------------------------
// Byte offsets of every region of a rank call's workspace; kge_rank_workspace_bytes is `total`.  The two
// directions never share a query-side buffer: they may run concurrently on two streams.  The fp32 tiled
// sweep's regions exist for tiled_supported models, the tensor-core regions for the models tc_supported
// admits at some table size.
struct RankLayout {
  size_t thr[2];               // [Q] thresholds: the target's own score
  size_t qvec[2];              // [Q][KQ][dp] query vectors of the tiled sweep
  size_t qscale[2];            // [Q] TransM scale theta[r]
  size_t cand;                 // [KC][num_ent][dp] candidate scratch (normalised / padded / realigned rows); unused
                               // by TransE on the tensor-core path when the fallback can read the table itself
  size_t a[2][2];              // [dir][0: high, 1: low] bf16 query operands [Q][Kp]
  size_t tau[2];               // [Q][4] band coefficients (centre, a, b, e) of tc_query_finish
  size_t tc_counts[2];         // [Q] certain counts of level 1 (+ the resolved pairs of level 2)
  size_t ctrl[2];              // [4] pair-list length, overflow, resolve-and-commit done counter (+ 1 unused)
  size_t list[2];              // [tc_list_capacity(Q)] (q << 32 | local candidate row)
  size_t b[2];                 // [0: high, 1: low] bf16 candidate operands [num_ent][Kp]
  size_t cn;                   // [num_ent] candidate norm bounds
  size_t cinv;                 // [num_ent] TransE: the canonical inverse norm of every candidate row
  size_t total;
};
RankLayout rank_layout(const kge_model_t* m, int64_t Q);

// ---- one rank call ----------------------------------------------------------------------------------
// A direction's CSR filter (global entity ids) and the targets it must not count.
struct RankFilter { const int64_t* ptr; const int64_t* idx; int64_t nnz; const int64_t* tgt; };

// dir 0: tail sweep (TAIL grouping, counts columns 0/1), dir 1: head sweep (HEAD grouping, columns 2/3).
struct RankCall {
  const kge_model_t* m;        // candidate-side tables, rows [row_lo, row_hi)
  const kge_model_t* mq;       // query-side tables
  const int64_t *qh, *qr, *qt;
  int64_t Q, nc, row_lo, row_hi;
  RankFilter filt[2];
  int32_t* counts;
  char* ws;
  RankLayout L;
  bool use_tiled, use_tc;
  template <class T> T* at(size_t off) const { return reinterpret_cast<T*>(ws + off); }
  float* thr(int dir) const { return at<float>(L.thr[dir]); }
};

// The stages, in the order kge_rank_1vsall enqueues them for a direction (all capture-safe: no host sync,
// no allocation):
//   prepare_candidates   once per call (tiled paths): candidate scratch and, with use_tc, the bf16 candidate
//                        operands shared by both directions
//   prepare_queries      thresholds thr[q], the tiled sweep's query vectors and, with use_tc, the tensor-core
//                        query operands and band coefficients; CP's per-direction candidate operands first
//   tc_sweep             level 1 of one direction, or of both (ndirs == 2, dir == 0) in one grid.z = 2 launch;
//                        dots: optional [Q][nc] raw accumulators of direction `dir` (tests)
//   tc_resolve_commit    use_tc, one launch: exact fp32 re-evaluation of the ambiguous pairs of level 1 and of the
//                        filter entries, then counts += tc_counts; or, when the pair list overflowed, the fp32
//                        tiled sweep of the direction and the filter corrections
//   resolve_pairs        without use_tc: exact fp32 re-evaluation of the filter entries (the filter corrections)
//   tiled_sweep          without use_tc: the fp32 sweep
int prepare_candidates(const RankCall& C, cudaStream_t st);
int prepare_queries(const RankCall& C, int dir, cudaStream_t st);
int tc_sweep(const RankCall& C, int dir, int ndirs, float* dots, cudaStream_t st);
int tc_resolve_commit(const RankCall& C, int dir, cudaStream_t st);
int resolve_pairs(const RankCall& C, int dir, cudaStream_t st);
int tiled_sweep(const RankCall& C, int dir, cudaStream_t st);

// Used by the preparation stages of kge_rank_tiled.cu.  src[k]: the fp32 candidate tables (row pitch m->dim);
// scratch: optional fp32 copy [KC][nc][dp] for the fp32 fallback sweep, written by the same kernel; cinv
// (TransE): optional [nc] inverse row norms, with which the fallback normalises the raw rows it stages.
int tc_prepare_candidates(const RankCall& C, const float* const src[2], float* scratch, float* cinv, cudaStream_t st);
struct TcQueryArgs;
TcQueryArgs tc_query_args(const RankCall& C, int dir);

// Measurement hook (KGE_RANK_PROFILE): CUDA events recorded immediately around the launch of a
// direction's main sweep kernel (tensor-core or fp32) on the stream it is launched on.
struct SweepProfile { cudaEvent_t beg = nullptr, end = nullptr; bool armed = false, valid = false; int ndirs = 1; };
SweepProfile* sweep_profile(int dir);
void tc_set_trace(long long* buf);

// A kernel launched with more dynamic shared memory than the default 48 KB must opt in first.
template <class Kernel>
int smem_optin(Kernel kernel, size_t smem) {
  if (smem > 40 * 1024)
    KGE_CUDA_OK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return KGE_OK;
}
}  // namespace kge
