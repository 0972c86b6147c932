// kge_score.cu — fused gather + score forward:  replaces model.forward(h, r, t)
// (pykg2vec/models/pairwise.py, pointwise.py; callers pykg2vec/utils/trainer.py:147-180).
//
// Mapping: one 8-lane group per triple (4 triples per warp, 32 per 256-thread CTA).
// Lane l reads the 16-byte chunks l, l+8, ... of every gathered row, so the 8 lanes
// of a group cover 128 contiguous bytes of a row per load instruction (one full
// cache line when the row is line-aligned), and a warp has 4 x (rows per triple)
// independent row streams in flight.  HBM-bound: rows*d*4 + 28 bytes per triple.
#include <cstdlib>

#include "kge_models.cuh"

namespace kge {

constexpr int kThreads = 256;
constexpr int kGroupsPerCta = kThreads / 8;

template <int MODEL, int VEC, int CHSEL>
__global__ void __launch_bounds__(kThreads, 2)  // <= 128 registers: at least 16 warps per SM in flight
score_fwd_kernel(ModelParams P, int grouping, const int64_t* __restrict__ h,
                 const int64_t* __restrict__ r, const int64_t* __restrict__ t, int64_t n,
                 float* __restrict__ out, int scratch_floats) {
  extern __shared__ float4 smem_f4[];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const int64_t g = (int64_t)blockIdx.x * kGroupsPerCta + (threadIdx.x >> 3);
  const bool valid = g < n;
  const int64_t gi = valid ? g : n - 1;  // idle groups shadow the last triple (shuffles stay full-warp)
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.tab, P.tab, P.tab, __ldg(h + gi), __ldg(r + gi), __ldg(t + gi));
  float s;
  if (grouping == KGE_GROUP_TAIL) s = score_group<MODEL, VEC, KGE_GROUP_TAIL, CHSEL>(R, P, lane, scratch);
  else s = score_group<MODEL, VEC, KGE_GROUP_HEAD, CHSEL>(R, P, lane, scratch);
  if (valid && lane == 0) out[g] = s;
}

// ---- TransE / TransM, large batches: persistent CTAs, rows staged in shared memory by cp.async --------
// The register-cached kernel above holds a triple's three rows in registers (84 of its 115 registers at
// d = 200), which caps it at 2 CTAs per SM that move in lock step through ids -> rows -> compute, so the
// row loads of a CTA are never in flight while it computes.  Here a
// CTA is persistent and software-pipelined: lane l of a group copies ITS chunks (l, l+8, ...) of the
// three rows of the NEXT triple into a shared-memory stage with 16-byte cp.async (LDGSTS: no registers
// are tied up, nothing waits), the ids of the triple after that are already in registers, and the current
// triple is evaluated from the other stage with exactly the two-pass arithmetic of trans_distance (CH = 0).
// A lane only ever reads what it copied itself, so there is no barrier anywhere in the loop.
KGE_DEV void cp_async16(void* smem_dst, const void* gsrc) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
KGE_DEV void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> KGE_DEV void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int MODEL, int GROUPING>
__global__ void __launch_bounds__(kThreads, 1)
score_fwd_staged_kernel(ModelParams P, const int64_t* __restrict__ h, const int64_t* __restrict__ r,
                        const int64_t* __restrict__ t, int64_t n, float* __restrict__ out, int64_t ntiles) {
  extern __shared__ float4 smem_f4[];
  const int lane = threadIdx.x & 7, grp = threadIdx.x >> 3;
  const int d = P.d, nch = d >> 2;                       // d % 4 == 0 (host checks)
  float4* const st0 = smem_f4 + (size_t)grp * 3 * nch;
  float4* const st1 = st0 + (size_t)kGroupsPerCta * 3 * nch;
  const float* const ent = P.tab[0];
  const float* const rel = P.tab[1];
  struct Ids { int64_t h, r, t; };
  auto load_ids = [&](int64_t tile) {
    Ids I;
    int64_t g = tile * kGroupsPerCta + grp;
    if (g >= n) g = n - 1;                               // idle groups shadow the last triple
    I.h = __ldg(h + g); I.r = __ldg(r + g); I.t = __ldg(t + g);
    return I;
  };
  auto issue = [&](float4* st, const Ids& I) {
    const float4* hp = reinterpret_cast<const float4*>(ent + (size_t)I.h * d);
    const float4* rp = reinterpret_cast<const float4*>(rel + (size_t)I.r * d);
    const float4* tp = reinterpret_cast<const float4*>(ent + (size_t)I.t * d);
    for (int c = lane; c < nch; c += 8) {
      cp_async16(st + c, hp + c);
      cp_async16(st + nch + c, rp + c);
      cp_async16(st + 2 * nch + c, tp + c);
    }
  };
  const int64_t stride = gridDim.x;
  int64_t tile = blockIdx.x;
  if (tile >= ntiles) return;
  Ids cur = load_ids(tile);
  issue(st0, cur);
  cp_async_commit();
  Ids nxt = cur;
  if (tile + stride < ntiles) nxt = load_ids(tile + stride);
  int buf = 0;
  for (; tile < ntiles; tile += stride, buf ^= 1) {
    float4* const mine = buf ? st1 : st0;
    const bool more = tile + stride < ntiles;
    if (more) issue(buf ? st0 : st1, nxt);               // rows of the next tile: in flight during this tile's math
    cp_async_commit();
    const Ids keep = cur;
    cur = nxt;
    if (tile + 2 * stride < ntiles) nxt = load_ids(tile + 2 * stride);   // ids two tiles ahead: off the critical path
    cp_async_wait<1>();                                  // this lane's copies of the current tile have landed
    auto fh = [&](int c) { return mine[c]; };
    auto fr = [&](int c) { return mine[nch + c]; };
    auto ft = [&](int c) { return mine[2 * nch + c]; };
    float s = trans_distance<GROUPING, 0>(fh, fr, ft, nch, lane, P.l1);
    if (MODEL == KGE_TRANSM) s = fmul(__ldg(P.tab[2] + keep.r), s);   // theta[r] * distance (pairwise.py:325-347)
    const int64_t g = tile * kGroupsPerCta + grp;
    if (g < n && lane == 0) out[g] = s;
  }
  cp_async_wait<0>();
}

int check_model(const kge_model_t* m) {
  if (!m) { set_error("model is NULL"); return KGE_EINVAL; }
  const int nt = num_tables(m->model);
  if (nt == 0) { set_error("unknown model id %d", m->model); return KGE_ENOTSUP; }
  if (m->dim <= 0 || m->rel_dim <= 0 || m->num_ent <= 0 || m->num_rel <= 0) {
    set_error("bad model geometry dim=%d rel_dim=%d num_ent=%lld num_rel=%lld", m->dim, m->rel_dim,
              (long long)m->num_ent, (long long)m->num_rel);
    return KGE_EINVAL;
  }
  for (int k = 0; k < nt; ++k)
    if (!m->tables[k]) { set_error("tables[%d] is NULL", k); return KGE_EINVAL; }
  if (m->model == KGE_ANALOGY && (m->dim % 2)) { set_error("ANALOGY needs an even hidden_size"); return KGE_EINVAL; }
  const bool free_rel_dim = m->model == KGE_TRANSR || m->model == KGE_SLM || m->model == KGE_NTN;
  if (!free_rel_dim && m->rel_dim != m->dim) {
    // TransD as written only broadcasts when ent_hidden_size == rel_hidden_size (pairwise.py:275-278)
    set_error("rel_dim (%d) must equal dim (%d) for this model", m->rel_dim, m->dim);
    return KGE_EINVAL;
  }
  return KGE_OK;
}

int model_vec(const kge_model_t* m) {
  const int nt = num_tables(m->model);
  if (m->model == KGE_TRANSM) return pick_vec(m, 2, m->dim);  // theta is a [R] vector, read as scalars
  if (m->model == KGE_ANALOGY) {  // half-width rows must keep the vector alignment too
    if (m->dim % 2) return 1;
    return pick_vec(m, nt, m->dim / 2);
  }
  if (m->model == KGE_HOLE) return (m->dim % 4 == 0) ? pick_vec(m, nt, m->dim) : 1;  // mirrored scalar reads
  if (m->model == KGE_SLM || m->model == KGE_NTN) return pick_vec(m, nt, m->dim, m->rel_dim);
  if (m->model == KGE_SME || m->model == KGE_SME_BL) return pick_vec(m, 2, m->dim);  // matrices: scalar reads
  if (m->model == KGE_CONVKB) return pick_vec(m, 3, m->dim);                          // c0 is one scalar
  return pick_vec(m, nt, m->dim, m->model == KGE_TRANSR ? m->rel_dim : 0);
}

}  // namespace kge

using namespace kge;

extern "C" int kge_score_fwd(const kge_model_t* m, int grouping, const int64_t* h, const int64_t* r,
                             const int64_t* t, int64_t n, float* scores, void* stream) {
  int rc = check_model(m);
  if (rc) return rc;
  if (n == 0) return KGE_OK;
  if (n < 0 || !h || !r || !t || !scores) { set_error("kge_score_fwd: bad arguments"); return KGE_EINVAL; }
  if (grouping != KGE_GROUP_TAIL && grouping != KGE_GROUP_HEAD) { set_error("bad grouping"); return KGE_EINVAL; }
  const ModelParams P = make_params(m, nullptr);
  const int vec = model_vec(m);
  const int sf = (int)group_scratch_floats(m);
  const size_t smem = (size_t)sf * kGroupsPerCta * sizeof(float);
  if (smem > 227 * 1024) {
    set_error("%s: embedding width too large for this model's per-group scratch (%zu B of shared memory)", "kge_score_fwd", smem);
    return KGE_ENOTSUP;
  }
  const unsigned grid = (unsigned)((n + kGroupsPerCta - 1) / kGroupsPerCta);
  cudaStream_t st = (cudaStream_t)stream;
  if ((m->model == KGE_TRANSE || m->model == KGE_TRANSM) && vec == 4 && m->dim % 4 == 0 && !getenv("KGE_SCORE_NO_STAGED")) {
    // large batches: persistent cp.async-staged kernel (one CTA per SM, two stages of 32 triples)
    const size_t stage_smem = (size_t)2 * kGroupsPerCta * 3 * (size_t)m->dim * sizeof(float);
    const int64_t ntiles = (n + kGroupsPerCta - 1) / kGroupsPerCta;
    if (stage_smem <= 227 * 1024 && ntiles >= 4 * (int64_t)sm_count()) {
      const unsigned pgrid = (unsigned)sm_count();
#define LAUNCH_STAGED(M)                                                                                   \
  do {                                                                                                     \
    if (grouping == KGE_GROUP_TAIL) {                                                                      \
      KGE_CUDA_OK(cudaFuncSetAttribute(score_fwd_staged_kernel<M, KGE_GROUP_TAIL>,                         \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_smem));     \
      score_fwd_staged_kernel<M, KGE_GROUP_TAIL><<<pgrid, kThreads, stage_smem, st>>>(P, h, r, t, n, scores, ntiles); \
    } else {                                                                                               \
      KGE_CUDA_OK(cudaFuncSetAttribute(score_fwd_staged_kernel<M, KGE_GROUP_HEAD>,                         \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)stage_smem));     \
      score_fwd_staged_kernel<M, KGE_GROUP_HEAD><<<pgrid, kThreads, stage_smem, st>>>(P, h, r, t, n, scores, ntiles); \
    }                                                                                                      \
  } while (0)
      if (m->model == KGE_TRANSE) LAUNCH_STAGED(KGE_TRANSE); else LAUNCH_STAGED(KGE_TRANSM);
#undef LAUNCH_STAGED
      KGE_CHECK_LAUNCH("score_fwd_staged_kernel");
      return KGE_OK;
    }
  }
  // distance models: the register-cache depth is a template parameter picked from the width
  // (TransD gathers six rows per triple: re-reading them from L1 at high occupancy beats caching
  //  the projected operands at <= 128 registers — 0.89 vs 0.78 of HBM peak measured — so CH = 0)
  int chsel = (is_distance_model(m->model) && m->model != KGE_TRANSD)
                  ? ch_select(m->model == KGE_TRANSR ? m->rel_dim : m->dim) : 0;
  if (const char* e = getenv("KGE_SCORE_CH")) {   // tuning aid (read per call): force the register-cache depth
    const int v = atoi(e);
    const int need = (((m->model == KGE_TRANSR ? m->rel_dim : m->dim) + 3) / 4 + 7) / 8;
    if (is_distance_model(m->model) && (v == 0 || ((v == 2 || v == 4 || v == 8) && v >= need))) chsel = v;
  }
#define LAUNCH(M, V, C)                                                                            \
  do {                                                                                             \
    if (smem > 40 * 1024)                                                                          \
      KGE_CUDA_OK(cudaFuncSetAttribute(score_fwd_kernel<M, V, C>,                                  \
                                       cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));   \
    score_fwd_kernel<M, V, C><<<grid, kThreads, smem, st>>>(P, grouping, h, r, t, n, scores, sf);  \
  } while (0)
#define CALL(M, V)                                                       \
  do {                                                                   \
    if (!is_distance_model(M)) { LAUNCH(M, V, 0); }                      \
    else if (chsel == 2) { LAUNCH(M, V, 2); }                            \
    else if (chsel == 4) { LAUNCH(M, V, 4); }                            \
    else if (chsel == 8) { LAUNCH(M, V, 8); }                            \
    else { LAUNCH(M, V, 0); }                                            \
  } while (0)
  KGE_DISPATCH_MODEL_VEC(m->model, vec, CALL);
#undef CALL
#undef LAUNCH
  KGE_CHECK_LAUNCH("score_fwd_kernel");
  return KGE_OK;
}
