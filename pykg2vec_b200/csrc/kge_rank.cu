// kge_rank.cu — 1-vs-all link-prediction rank counts: replaces Evaluator.test
// (pykg2vec/utils/evaluator.py:309-334) together with the Python rank walk of
// MetricCalculator.get_tail_rank/get_head_rank (evaluator.py:70-123).
//
// Instead of materialising N scores, sorting them (topk k=N), copying the ids to
// the host and walking the list, each query's rank is COUNTED on the device:
//   raw      = #{e in [row_lo,row_hi) : score_e < score_target}
//   filtered = raw - #{e in filter(q), e != target : score_e < score_target}
// Scores use exactly the arithmetic of kge_score_fwd (DESIGN.md §3), so counts of
// disjoint row shards add up to the global rank.
//
// Two sweep implementations:
//   * gather sweep (all models): the fused gather+score group function evaluated
//     over (query, candidate) pairs; one CTA = one query x 512 consecutive candidates.
//   * tiled sweep (kge_rank_tiled.cu; TransE/TransM, DistMult/CP, ComplEx, RotatE):
//     query vectors and candidate rows staged in shared memory by bulk-async copies,
//     register-tiled pair evaluation, FMA-pipe bound.
#include "kge_models.cuh"
#include "kge_rank.cuh"
#include "kge_rank_resolve.cuh"

namespace kge {

constexpr int kThreads = 256;
constexpr int kGroupsPerCta = kThreads / 8;
constexpr int kSweepIters = 16;
constexpr int kCandsPerCta = kGroupsPerCta * kSweepIters;

template <int MODEL, int VEC, int GROUPING>
__global__ void __launch_bounds__(kThreads)
sweep_gather_kernel(ModelParams P, const int64_t* __restrict__ qh, const int64_t* __restrict__ qr,
                    const int64_t* __restrict__ qt, const float* __restrict__ thr, int64_t nc,
                    int32_t* __restrict__ counts, int col, int scratch_floats) {
  extern __shared__ float4 smem_f4[];
  __shared__ int block_cnt;
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const int64_t q = blockIdx.y;
  const int64_t h = __ldg(qh + q), r = __ldg(qr + q), t = __ldg(qt + q);
  const float th = __ldg(thr + q);
  if (threadIdx.x == 0) block_cnt = 0;
  __syncthreads();
  const int64_t base = (int64_t)blockIdx.x * kCandsPerCta;
  int cnt = 0;
  for (int it = 0; it < kSweepIters; ++it) {
    const int64_t e = base + it * kGroupsPerCta + grp;
    const bool valid = e < nc;
    const int64_t ei = valid ? e : nc - 1;
    TripleRows R;
    if (GROUPING == KGE_GROUP_TAIL) resolve_rows<MODEL>(R, P, P.qtab, P.tab, P.qtab, h, r, ei);
    else resolve_rows<MODEL>(R, P, P.tab, P.qtab, P.qtab, ei, r, t);
    const float s = score_group<MODEL, VEC, GROUPING>(R, P, lane, scratch);
    cnt += (valid && s < th) ? 1 : 0;
  }
  if (lane == 0 && cnt) atomicAdd(&block_cnt, cnt);
  __syncthreads();
  if (threadIdx.x == 0 && block_cnt) {
    atomicAdd(counts + q * 4 + col, block_cnt);
    atomicAdd(counts + q * 4 + col + 1, block_cnt);
  }
}

// thresholds: the target's own score, evaluated on the query-side tables
template <int MODEL, int VEC, int GROUPING>
__global__ void __launch_bounds__(kThreads)
threshold_kernel(ModelParams P, const int64_t* __restrict__ qh, const int64_t* __restrict__ qr,
                 const int64_t* __restrict__ qt, int64_t Q, float* __restrict__ thr, int scratch_floats) {
  extern __shared__ float4 smem_f4[];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * kGroupsPerCta + (threadIdx.x >> 3);
  const bool valid = g < Q;
  const int64_t gi = valid ? g : Q - 1;
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.qtab, P.qtab, P.qtab, __ldg(qh + gi), __ldg(qr + gi), __ldg(qt + gi));
  const float s = score_group<MODEL, VEC, GROUPING>(R, P, lane, scratch);
  if (valid && lane == 0) thr[g] = s;
}

// the filter pass of the gather and fp32 paths: exact re-evaluation of the filter entries (kge_rank_resolve.cuh)
template <int MODEL, int VEC, int GROUPING>
__global__ void __launch_bounds__(kResolveThreads)
resolve_pairs_kernel(const __grid_constant__ ModelParams P, const __grid_constant__ ResolveArgs A) {
  extern __shared__ float4 smem_f4[];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * A.scratch_floats;
  resolve_items<MODEL, VEC, GROUPING>(P, A, 0, scratch);
}

SweepProfile* sweep_profile(int dir) {
  static thread_local SweepProfile prof[2];
  return &prof[dir & 1];
}

int check_model(const kge_model_t* m);
int model_vec(const kge_model_t* m);

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

RankLayout rank_layout(const kge_model_t* m, int64_t Q) {
  RankLayout L = {};
  const size_t q = (size_t)Q;
  L.thr[0] = 0;
  L.thr[1] = q * sizeof(float);
  size_t o = align_up(2 * q * sizeof(float), 256);
  auto take = [&o](size_t bytes) { const size_t at = o; o += align_up(bytes, 256); return at; };
  if (tiled_supported(m)) {
    const size_t dp = (size_t)rank_dp(m), kq = (size_t)rank_kq(m->model);
    for (int d = 0; d < 2; ++d) L.qvec[d] = take(q * kq * dp * sizeof(float));
    for (int d = 0; d < 2; ++d) L.qscale[d] = take(q * sizeof(float));
    // always reserved: the alignment of the tables is only known at call time
    L.cand = take(kq * (size_t)m->num_ent * dp * sizeof(float));
    if (tc_supported(m, (int64_t)1 << 20)) {   // model-level support (the row count is only known per call)
      const size_t Kp = (size_t)tc_kp(m);
      for (int d = 0; d < 2; ++d) {
        for (int k = 0; k < 2; ++k) L.a[d][k] = take(q * Kp * 2);
        L.tau[d] = take(q * 4 * sizeof(float));
        L.tc_counts[d] = take(q * sizeof(int32_t));
        L.ctrl[d] = take(256);
        L.list[d] = take((size_t)tc_list_capacity(Q) * 8);
      }
      for (int k = 0; k < 2; ++k) L.b[k] = take((size_t)m->num_ent * Kp * 2);
      L.cn = take((size_t)m->num_ent * sizeof(float));
      if (m->model == KGE_TRANSE) L.cinv = take((size_t)m->num_ent * sizeof(float));
    }
  }
  L.total = o;
  return L;
}

GroupArgs group_args(const RankCall& C) {
  GroupArgs G;
  G.P = make_params(C.m, C.mq);
  G.vec = model_vec(C.m);
  const int vq = model_vec(C.mq);
  if (vq < G.vec) G.vec = vq;
  G.sf = (int)group_scratch_floats(C.m);
  G.smem = (size_t)G.sf * kGroupsPerCta * sizeof(float);
  return G;
}

// thresholds of the gather path (the tiled paths compute them in prepare_queries)
static int gather_thresholds(const RankCall& C, int dir, cudaStream_t st) {
  const GroupArgs G = group_args(C);
  decltype(&threshold_kernel<KGE_TRANSE, 4, KGE_GROUP_TAIL>) kernel;
#define PICK(M, V) kernel = dir == 0 ? threshold_kernel<M, V, KGE_GROUP_TAIL> : threshold_kernel<M, V, KGE_GROUP_HEAD>
  KGE_DISPATCH_MODEL_VEC(C.m->model, G.vec, PICK);
#undef PICK
  const int rc = smem_optin(kernel, G.smem);
  if (rc) return rc;
  kernel<<<(unsigned)((C.Q + kGroupsPerCta - 1) / kGroupsPerCta), kThreads, G.smem, st>>>(G.P, C.qh, C.qr, C.qt, C.Q,
                                                                                          C.thr(dir), G.sf);
  KGE_CHECK_LAUNCH("threshold_kernel");
  return KGE_OK;
}

static int gather_sweep(const RankCall& C, int dir, cudaStream_t st) {
  const GroupArgs G = group_args(C);
  decltype(&sweep_gather_kernel<KGE_TRANSE, 4, KGE_GROUP_TAIL>) kernel;
#define PICK(M, V) kernel = dir == 0 ? sweep_gather_kernel<M, V, KGE_GROUP_TAIL> : sweep_gather_kernel<M, V, KGE_GROUP_HEAD>
  KGE_DISPATCH_MODEL_VEC(C.m->model, G.vec, PICK);
#undef PICK
  const int rc = smem_optin(kernel, G.smem);
  if (rc) return rc;
  const dim3 grid((unsigned)((C.nc + kCandsPerCta - 1) / kCandsPerCta), (unsigned)C.Q);
  kernel<<<grid, kThreads, G.smem, st>>>(G.P, C.qh, C.qr, C.qt, C.thr(dir), C.nc, C.counts, 2 * dir, G.sf);
  KGE_CHECK_LAUNCH("sweep_gather_kernel");
  return KGE_OK;
}

ResolveArgs resolve_args(const RankCall& C, int dir) {
  ResolveArgs A;
  A.qh = C.qh; A.qr = C.qr; A.qt = C.qt; A.thr = C.thr(dir);
  A.list = C.use_tc ? C.at<unsigned long long>(C.L.list[dir]) : nullptr;
  A.ctrl = C.use_tc ? C.at<unsigned>(C.L.ctrl[dir]) : nullptr;
  A.cap = tc_list_capacity(C.Q);
  A.tc_counts = C.use_tc ? C.at<int32_t>(C.L.tc_counts[dir]) : nullptr;
  A.F = C.filt[dir];
  A.Q = C.Q; A.row_lo = C.row_lo; A.row_hi = C.row_hi;
  A.counts = C.counts; A.col = 2 * dir;
  A.scratch_floats = (int)group_scratch_floats(C.m);
  return A;
}

int resolve_pairs(const RankCall& C, int dir, cudaStream_t st) {
  const RankFilter& F = C.filt[dir];
  if (!(F.ptr && F.idx && F.nnz > 0)) return KGE_OK;
  const GroupArgs G = group_args(C);
  decltype(&resolve_pairs_kernel<KGE_TRANSE, 4, KGE_GROUP_TAIL>) kernel;
#define PICK(M, V) kernel = dir == 0 ? resolve_pairs_kernel<M, V, KGE_GROUP_TAIL> : resolve_pairs_kernel<M, V, KGE_GROUP_HEAD>
  KGE_DISPATCH_MODEL_VEC(C.m->model, G.vec, PICK);
#undef PICK
  const int rc = smem_optin(kernel, G.smem);
  if (rc) return rc;
  // one group per entry
  const unsigned grid = (unsigned)((F.nnz + kResolveGroups - 1) / kResolveGroups);
  kernel<<<grid, kResolveThreads, G.smem, st>>>(G.P, resolve_args(C, dir));
  KGE_CHECK_LAUNCH("resolve_pairs_kernel");
  return KGE_OK;
}

// Fork/join helper: the head-direction chain of a rank call runs on a side stream so that its
// short preparation / filter kernels overlap the other direction's sweep (and fill the idle
// SMs of its last wave); with the tensor-core sweep the two query preparations run on the two side
// streams beside the candidate preparation.  Streams and events are created lazily, once per host
// thread and device; event record / wait are capture-safe, so the pattern also works inside a CUDA
// graph capture.
struct SideStream {
  cudaStream_t stream = nullptr, stream2 = nullptr;
  cudaEvent_t fork = nullptr, join = nullptr, mid = nullptr, mid2 = nullptr, fork2 = nullptr;
  int device = -1;
};
static int side_stream(SideStream** out) {
  static thread_local SideStream ss[16];
  int dev = 0;
  KGE_CUDA_OK(cudaGetDevice(&dev));
  SideStream& s = ss[dev & 15];
  if (!s.stream) {
    KGE_CUDA_OK(cudaStreamCreateWithFlags(&s.stream, cudaStreamNonBlocking));
    KGE_CUDA_OK(cudaStreamCreateWithFlags(&s.stream2, cudaStreamNonBlocking));
    KGE_CUDA_OK(cudaEventCreateWithFlags(&s.fork, cudaEventDisableTiming));
    KGE_CUDA_OK(cudaEventCreateWithFlags(&s.join, cudaEventDisableTiming));
    KGE_CUDA_OK(cudaEventCreateWithFlags(&s.mid, cudaEventDisableTiming));
    KGE_CUDA_OK(cudaEventCreateWithFlags(&s.mid2, cudaEventDisableTiming));
    KGE_CUDA_OK(cudaEventCreateWithFlags(&s.fork2, cudaEventDisableTiming));
    s.device = dev;
  }
  *out = &s;
  return KGE_OK;
}

static RankCall make_call(const kge_model_t* m, const kge_model_t* mq, int64_t row_lo, int64_t row_hi,
                          const int64_t* qh, const int64_t* qr, const int64_t* qt, int64_t Q, int32_t* counts,
                          void* workspace) {
  RankCall C;
  C.m = m; C.mq = mq; C.qh = qh; C.qr = qr; C.qt = qt;
  C.Q = Q; C.nc = row_hi - row_lo; C.row_lo = row_lo; C.row_hi = row_hi;
  C.filt[0] = C.filt[1] = RankFilter{nullptr, nullptr, 0, nullptr};
  C.counts = counts; C.ws = reinterpret_cast<char*>(workspace);
  C.L = rank_layout(m, Q);
  C.use_tiled = C.use_tc = false;
  return C;
}

}  // namespace kge

using namespace kge;

extern "C" int64_t kge_rank_workspace_bytes(const kge_model_t* m, int64_t Q) {
  if (!m || Q < 0) return 0;
  return (int64_t)rank_layout(m, Q).total;
}

extern "C" int kge_rank_1vsall(const kge_model_t* m, const kge_model_t* mq, int64_t row_lo,
                               int64_t row_hi, const int64_t* qh, const int64_t* qr,
                               const int64_t* qt, const int64_t* tgt_h, const int64_t* tgt_t,
                               int64_t Q, const int64_t* filt_t_ptr, const int64_t* filt_t_idx,
                               int64_t filt_t_nnz, const int64_t* filt_h_ptr,
                               const int64_t* filt_h_idx, int64_t filt_h_nnz, int32_t* counts,
                               void* workspace, int64_t workspace_bytes, int flags, void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (!mq) mq = m;
  rc = check_model(mq);
  if (rc) return rc;
  if (mq->model != m->model || mq->dim != m->dim || mq->rel_dim != m->rel_dim) {
    set_error("kge_rank_1vsall: m and mq describe different models"); return KGE_EINVAL;
  }
  if (Q == 0) return KGE_OK;
  if (Q < 0 || !qh || !qr || !qt || !counts || !workspace || row_lo < 0 || row_hi <= row_lo ||
      row_hi - row_lo > m->num_ent) {
    set_error("kge_rank_1vsall: bad arguments"); return KGE_EINVAL;
  }
  if (Q > 65535) { set_error("kge_rank_1vsall: Q=%lld > 65535, batch the queries", (long long)Q); return KGE_EINVAL; }
  if (workspace_bytes < kge_rank_workspace_bytes(m, Q)) { set_error("workspace too small"); return KGE_EWORKSPACE; }
  if (group_scratch_floats(m) * kGroupsPerCta * sizeof(float) > 227 * 1024) {
    set_error("kge_rank_1vsall: embedding width too large for this model's scratch"); return KGE_ENOTSUP;
  }
  RankCall C = make_call(m, mq, row_lo, row_hi, qh, qr, qt, Q, counts, workspace);
  C.filt[0] = RankFilter{filt_t_ptr, filt_t_idx, filt_t_nnz, tgt_t ? tgt_t : qt};
  C.filt[1] = RankFilter{filt_h_ptr, filt_h_idx, filt_h_nnz, tgt_h ? tgt_h : qh};
  C.use_tiled = !(flags & KGE_RANK_FORCE_GATHER) && tiled_supported(m);
  C.use_tc = C.use_tiled && !(flags & KGE_RANK_NO_TC) && tc_supported(m, C.nc);
  const cudaStream_t main_st = (cudaStream_t)stream;
  for (int d = 0; d < 2; ++d) {
    SweepProfile* sp = sweep_profile(d);
    sp->armed = (flags & KGE_RANK_PROFILE) != 0;
    sp->valid = false;
    sp->ndirs = 1;
    if (sp->armed && !sp->beg) {
      KGE_CUDA_OK(cudaEventCreate(&sp->beg));
      KGE_CUDA_OK(cudaEventCreate(&sp->end));
    }
  }
  const bool run[2] = {!(flags & KGE_RANK_HEAD_ONLY), !(flags & KGE_RANK_TAIL_ONLY)};
  // (CP / SimplE refill one shared candidate scratch per direction: their directions stay serial)
  const bool dirs_independent = m->model != KGE_CP && !is_simple(m->model);
  const bool two_streams = run[0] && run[1] && C.use_tiled && dirs_independent && !(flags & KGE_RANK_SINGLE_STREAM);
  // Both directions on the tensor cores: the two query preparations run on the two side streams from the start,
  // beside the candidate preparation (they read none of its outputs), ONE launch sweeps both directions (grid.z = 2:
  // same candidate operands; the launch / pipeline-ramp / drain overhead — a third of a 25 us sweep at the
  // FB15k-237 shape — is paid once and the tile units of both directions balance over the SMs), then the two
  // resolve-and-commit launches run side by side.
  const bool tc_both = C.use_tc && two_streams;
  SideStream* side = nullptr;
  auto fork = [&]() {
    KGE_CUDA_OK(cudaEventRecord(side->fork, main_st));
    KGE_CUDA_OK(cudaStreamWaitEvent(side->stream, side->fork, 0));
    if (tc_both) KGE_CUDA_OK(cudaStreamWaitEvent(side->stream2, side->fork, 0));
    return KGE_OK;
  };
  if (two_streams) {
    rc = side_stream(&side);
    if (rc) return rc;
  }
  if (tc_both && (rc = fork())) return rc;
  if (C.use_tiled) {
    rc = prepare_candidates(C, main_st);
    if (rc) return rc;
  }
  if (two_streams && !tc_both && (rc = fork())) return rc;   // the fp32 sweeps read the prepared candidates
  auto stream_of = [&](int dir) { return (two_streams && dir == 1) ? side->stream : main_st; };
  auto resolve_and_sweep = [&](int dir) {
    if (C.use_tc) return tc_resolve_commit(C, dir, stream_of(dir));
    const int r = resolve_pairs(C, dir, stream_of(dir));
    if (r) return r;
    return C.use_tiled ? tiled_sweep(C, dir, stream_of(dir)) : gather_sweep(C, dir, stream_of(dir));
  };
  for (int dir = 0; dir < 2; ++dir) {
    if (!run[dir]) continue;
    const cudaStream_t prep_st = tc_both ? (dir == 0 ? side->stream : side->stream2) : stream_of(dir);
    rc = C.use_tiled ? prepare_queries(C, dir, prep_st) : gather_thresholds(C, dir, prep_st);
    if (rc) return rc;
    if (tc_both) continue;
    if (C.use_tc) {
      rc = tc_sweep(C, dir, 1, nullptr, stream_of(dir));
      if (rc) return rc;
    }
    rc = resolve_and_sweep(dir);
    if (rc) return rc;
  }
  if (tc_both) {
    KGE_CUDA_OK(cudaEventRecord(side->mid, side->stream));
    KGE_CUDA_OK(cudaEventRecord(side->mid2, side->stream2));
    KGE_CUDA_OK(cudaStreamWaitEvent(main_st, side->mid, 0));
    KGE_CUDA_OK(cudaStreamWaitEvent(main_st, side->mid2, 0));
    rc = tc_sweep(C, 0, 2, nullptr, main_st);
    if (rc) return rc;
    KGE_CUDA_OK(cudaEventRecord(side->fork2, main_st));
    KGE_CUDA_OK(cudaStreamWaitEvent(side->stream, side->fork2, 0));
    for (int dir = 0; dir < 2; ++dir) {
      rc = resolve_and_sweep(dir);
      if (rc) return rc;
    }
  }
  if (two_streams) {
    KGE_CUDA_OK(cudaEventRecord(side->join, side->stream));
    KGE_CUDA_OK(cudaStreamWaitEvent(main_st, side->join, 0));
  }
  return KGE_OK;
}

// Test / measurement aid for the tensor-core level of one direction: raw accumulators and the band
// (see include/kge_b200.h).  Runs the stages of kge_rank_1vsall for that direction without filters.
extern "C" int kge_rank_tc_probe(const kge_model_t* m, const kge_model_t* mq, int64_t row_lo, int64_t row_hi,
                                 const int64_t* qh, const int64_t* qr, const int64_t* qt, int64_t Q, int direction,
                                 float* dots, float* tau, int32_t* counts, void* workspace, int64_t workspace_bytes,
                                 void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (!mq) mq = m;
  rc = check_model(mq);
  if (rc) return rc;
  if (Q <= 0 || Q > 65535 || !qh || !qr || !qt || !counts || !workspace || row_lo < 0 || row_hi <= row_lo ||
      row_hi - row_lo > m->num_ent || (direction != 0 && direction != 1)) {
    set_error("kge_rank_tc_probe: bad arguments"); return KGE_EINVAL;
  }
  if (!tiled_supported(m) || !tc_supported(m, row_hi - row_lo)) {
    set_error("kge_rank_tc_probe: no tensor-core sweep for this model / table size"); return KGE_ENOTSUP;
  }
  if (workspace_bytes < kge_rank_workspace_bytes(m, Q)) { set_error("workspace too small"); return KGE_EWORKSPACE; }
  const cudaStream_t st = (cudaStream_t)stream;
  RankCall C = make_call(m, mq, row_lo, row_hi, qh, qr, qt, Q, counts, workspace);
  C.use_tiled = C.use_tc = true;
  if ((rc = prepare_candidates(C, st)) || (rc = prepare_queries(C, direction, st)) ||
      (rc = tc_sweep(C, direction, 1, dots, st)))
    return rc;
  if (tau) {   // [Q][4] band coefficients, then the nc candidate norm bounds
    KGE_CUDA_OK(cudaMemcpyAsync(tau, C.ws + C.L.tau[direction], (size_t)Q * 4 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    KGE_CUDA_OK(cudaMemcpyAsync(tau + (size_t)Q * 4, C.ws + C.L.cn, (size_t)C.nc * sizeof(float), cudaMemcpyDeviceToDevice, st));
  }
  return tc_resolve_commit(C, direction, st);
}

extern "C" int kge_rank_last_sweep_directions(void) {
  SweepProfile* sp = sweep_profile(0);
  return sp->valid ? sp->ndirs : 0;
}

extern "C" int kge_rank_last_sweep_ms(int direction, float* ms) {
  if (!ms || (direction != 0 && direction != 1)) { set_error("kge_rank_last_sweep_ms: bad arguments"); return KGE_EINVAL; }
  SweepProfile* sp = sweep_profile(direction);
  if (!sp->valid) { set_error("kge_rank_last_sweep_ms: the last kge_rank_1vsall of this thread did not profile direction %d", direction); return KGE_EINVAL; }
  KGE_CUDA_OK(cudaEventSynchronize(sp->end));
  KGE_CUDA_OK(cudaEventElapsedTime(ms, sp->beg, sp->end));
  return KGE_OK;
}

// Measurement aid: clock64 stamps of CTA (0,0) of the following tc_sweep_kernel launches are written to
// buf[3 roles][64] (device memory; NULL switches it off).  Roles: 0 TMA producer (slot 0 start, then one
// per acquired stage), 1 consumer warpgroup start (warp 4), 2 epilogue begin / end per tile (warp 4);
// slot 63 of role 2: kernel entry, slot 62: cycles at the exit of CTA 0.
extern "C" int kge_debug_set_tc_trace(long long* buf) {
  tc_set_trace(buf);
  return KGE_OK;
}
