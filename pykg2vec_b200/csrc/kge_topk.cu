// kge_topk.cu — C-ABI launchers of batched top-k link prediction (kernels: kge_topk.cuh; declarations and
// reference citations: include/kge_b200.h).  Each call loops over chunks of at most topk_chunk_rows queries:
// producer launch into the workspace, then one select launch.  No host sync and no allocation inside the loop.
#include "kge_rank.cuh"
#include "kge_topk.cuh"

namespace kge {

int check_model(const kge_model_t* m);
int model_vec(const kge_model_t* m);

namespace {

int check_topk(const char* fn, int64_t Q, int64_t n, int32_t k, const int64_t* fptr, const int64_t* fidx,
               int64_t fnnz) {
  if (k < 1 || k > kTopkMaxK) { set_error("%s: k=%d outside [1, %d]", fn, (int)k, kTopkMaxK); return KGE_EINVAL; }
  if (Q < 0) { set_error("%s: Q=%lld < 0", fn, (long long)Q); return KGE_EINVAL; }
  if (n < 1 || n > (1ll << 30)) { set_error("%s: %lld candidates", fn, (long long)n); return KGE_EINVAL; }
  if (fnnz < 0 || (fnnz > 0 && (!fptr || !fidx))) { set_error("%s: bad filter", fn); return KGE_EINVAL; }
  if (topk_select_plan(n).smem == 0) {
    set_error("%s: %lld candidates: the filter bitmap exceeds shared memory", fn, (long long)n);
    return KGE_ENOTSUP;
  }
  return KGE_OK;
}

int check_outputs(const char* fn, int64_t* ids, float* scores, void* ws, int64_t ws_bytes, int64_t Q, int64_t n,
                  int32_t k) {
  if (!ids || !scores || !ws) { set_error("%s: null output or workspace", fn); return KGE_EINVAL; }
  if (ws_bytes < kge_topk_workspace_bytes(Q, n, k)) { set_error("%s: workspace too small", fn); return KGE_EWORKSPACE; }
  return KGE_OK;
}

int launch_select(const float* scores, int64_t rows, int64_t n, int32_t k, bool descending, const int64_t* fptr,
                  const int64_t* fidx, int64_t* ids, float* out_scores, cudaStream_t st) {
  const TopkSelectPlan plan = topk_select_plan(n);
  const TopkSelectArgs A{scores, n, (int)k, descending, fptr, fidx, ids, out_scores};
  auto kernel = plan.row_in_smem ? topk_select_kernel<true> : topk_select_kernel<false>;
  if (int rc = smem_optin(kernel, plan.smem)) return rc;
  kernel<<<(unsigned)rows, kTopkThreads, plan.smem, st>>>(A);
  KGE_CHECK_LAUNCH("topk_select_kernel");
  return KGE_OK;
}

}  // namespace
}  // namespace kge

using namespace kge;

extern "C" int64_t kge_topk_workspace_bytes(int64_t Q, int64_t n_cand, int32_t k) {
  if (Q < 0 || n_cand < 1 || k < 1 || k > kTopkMaxK) return 0;
  const int64_t rows = topk_chunk_rows(Q > 0 ? Q : 1, n_cand);
  return (rows * n_cand * (int64_t)sizeof(float) + 255) / 256 * 256;
}

extern "C" int kge_topk_1vsall(const kge_model_t* m, int32_t target, const int64_t* qh, const int64_t* qr,
                               const int64_t* qt, int64_t Q, int32_t k, const int64_t* filt_ptr,
                               const int64_t* filt_idx, int64_t filt_nnz, int64_t* out_ids, float* out_scores,
                               void* workspace, int64_t workspace_bytes, void* stream) {
  const char* fn = "kge_topk_1vsall";
  int rc = check_model(m);
  if (rc) return rc;
  if (target < 0 || target > 2) { set_error("%s: target %d is not 0 (tail), 1 (head) or 2 (relation)", fn, (int)target); return KGE_EINVAL; }
  const int64_t n = target == 2 ? m->num_rel : m->num_ent;
  if ((rc = check_topk(fn, Q, n, k, filt_ptr, filt_idx, filt_nnz))) return rc;
  if (Q == 0) return KGE_OK;
  if ((target != 1 && !qh) || (target != 2 && !qr) || (target != 0 && !qt)) { set_error("%s: null query ids", fn); return KGE_EINVAL; }
  if ((rc = check_outputs(fn, out_ids, out_scores, workspace, workspace_bytes, Q, n, k))) return rc;
  const size_t smem = group_scratch_floats(m) * kTopkGroups * sizeof(float);
  if (smem > 227 * 1024) { set_error("%s: embedding width too large for this model's scratch", fn); return KGE_ENOTSUP; }
  const ModelParams P = make_params(m, nullptr);
  const int sf = (int)group_scratch_floats(m);
  decltype(&topk_store_kernel<KGE_TRANSE, 4, 0>) kernel;
#define PICK(M, V) kernel = target == 0 ? topk_store_kernel<M, V, 0> : (target == 1 ? topk_store_kernel<M, V, 1> : topk_store_kernel<M, V, 2>)
  KGE_DISPATCH_MODEL_VEC(m->model, model_vec(m), PICK);
#undef PICK
  if ((rc = smem_optin(kernel, smem))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const bool filtered = filt_ptr && filt_idx && filt_nnz > 0;
  float* block = reinterpret_cast<float*>(workspace);
  const int64_t chunk = topk_chunk_rows(Q, n);
  for (int64_t q0 = 0; q0 < Q; q0 += chunk) {
    const int64_t rows = Q - q0 < chunk ? Q - q0 : chunk;
    const dim3 grid((unsigned)((n + kTopkCandsPerCta - 1) / kTopkCandsPerCta), (unsigned)rows);
    kernel<<<grid, kTopkThreads, smem, st>>>(P, qh ? qh + q0 : nullptr, qr ? qr + q0 : nullptr,
                                             qt ? qt + q0 : nullptr, n, block, sf);
    KGE_CHECK_LAUNCH("topk_store_kernel");
    if ((rc = launch_select(block, rows, n, k, false, filtered ? filt_ptr + q0 : nullptr, filt_idx,
                            out_ids + q0 * k, out_scores + q0 * k, st)))
      return rc;
  }
  return KGE_OK;
}

extern "C" int kge_proj_topk(const float* x, const float* ent, const float* bias, int64_t Q, int64_t N,
                             int32_t width, int32_t k, const int64_t* filt_ptr, const int64_t* filt_idx,
                             int64_t filt_nnz, int64_t* out_ids, float* out_scores, void* workspace,
                             int64_t workspace_bytes, void* stream) {
  const char* fn = "kge_proj_topk";
  if (!x || !ent) { set_error("%s: null x or ent", fn); return KGE_EINVAL; }
  if (width < 1) { set_error("%s: width=%d", fn, (int)width); return KGE_EINVAL; }
  int rc = check_topk(fn, Q, N, k, filt_ptr, filt_idx, filt_nnz);
  if (rc) return rc;
  if (Q == 0) return KGE_OK;
  if ((rc = check_outputs(fn, out_ids, out_scores, workspace, workspace_bytes, Q, N, k))) return rc;
  const cudaStream_t st = (cudaStream_t)stream;
  const bool filtered = filt_ptr && filt_idx && filt_nnz > 0;
  float* block = reinterpret_cast<float*>(workspace);
  const int64_t chunk = topk_chunk_rows(Q, N);
  for (int64_t q0 = 0; q0 < Q; q0 += chunk) {
    const int64_t rows = Q - q0 < chunk ? Q - q0 : chunk;
    // the forward's own launch (same tile choice, same bits as kge_proj_rank compares)
    if ((rc = kge_proj_tail_fwd(x + q0 * width, ent, bias, rows, N, width, block, stream))) return rc;
    if ((rc = launch_select(block, rows, N, k, true, filtered ? filt_ptr + q0 : nullptr, filt_idx,
                            out_ids + q0 * k, out_scores + q0 * k, st)))
      return rc;
  }
  return KGE_OK;
}
