// tests/emu/emu_topk.cpp — TEST INFRASTRUCTURE.  Runs the batched top-k kernels of pykg2vec_b200/csrc/kge_topk.cuh
// (the kernel-model score producer and the row selection) on the host, CUDA thread by CUDA thread
// (tests/emu/cuda_runtime.h), with the launch geometry and the shared-memory plan of the C-ABI launchers in
// kge_topk.cu (tests/test_emu_topk.py).  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include "cuda_runtime.h"

// shared-memory atomic the selection's filter bitmap uses (not part of the common emulation header)
inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }

#include "kge_topk.cuh"

namespace cuda_emu {
thread_local dim3 t_threadIdx, t_blockIdx;
dim3 g_blockDim, g_gridDim;
BlockCtx* g_block = nullptr;
std::mutex g_atomic_mu;
}  // namespace cuda_emu

namespace kge {  // host-side symbols kge_common.cuh declares (defined in kge_abi.cu in the product)
void set_error(const char*, ...) {}
int cuda_fail(cudaError_t, const char*) { return KGE_ECUDA; }
void count_launch(int) {}
int sm_count() { return 132; }
int num_tables(int) { return 0; }
}  // namespace kge

using namespace kge;

extern "C" {

// the select launch of kge_topk.cu for `rows` rows; returns whether the row was kept in shared memory
int emu_topk_select(const float* scores, int64_t rows, int64_t n, int k, int descending, const int64_t* fptr,
                    const int64_t* fidx, int64_t* ids, float* out) {
  const TopkSelectPlan plan = topk_select_plan(n);
  if (plan.smem == 0 || plan.smem > kTopkEmuSmem) return -1;
  const TopkSelectArgs A{scores, n, k, descending != 0, fptr, fidx, ids, out};
  if (plan.row_in_smem) cuda_emu::launch(dim3((unsigned)rows), dim3(kTopkThreads), [&] { topk_select_kernel<true>(A); });
  else cuda_emu::launch(dim3((unsigned)rows), dim3(kTopkThreads), [&] { topk_select_kernel<false>(A); });
  return plan.row_in_smem ? 1 : 0;
}

// the producer launch of kge_topk_1vsall for Q queries: out [Q, n]
int emu_topk_store(const kge_model_t* m, int target, int vec, const int64_t* qh, const int64_t* qr,
                   const int64_t* qt, int64_t Q, float* out) {
  const ModelParams P = make_params(m, nullptr);
  const int sf = (int)group_scratch_floats(m);
  if ((size_t)sf * kTopkGroups * sizeof(float) > kTopkEmuStoreSmem) return -2;
  const int64_t n = target == 2 ? m->num_rel : m->num_ent;
  const dim3 grid((unsigned)((n + kTopkCandsPerCta - 1) / kTopkCandsPerCta), (unsigned)Q);
#define CALL(M, V)                                                                                                \
  do {                                                                                                            \
    if (target == 0) cuda_emu::launch(grid, dim3(kTopkThreads), [&] { topk_store_kernel<M, V, 0>(P, qh, qr, qt, n, out, sf); }); \
    else if (target == 1) cuda_emu::launch(grid, dim3(kTopkThreads), [&] { topk_store_kernel<M, V, 1>(P, qh, qr, qt, n, out, sf); }); \
    else cuda_emu::launch(grid, dim3(kTopkThreads), [&] { topk_store_kernel<M, V, 2>(P, qh, qr, qt, n, out, sf); }); \
  } while (0)
  KGE_DISPATCH_MODEL_VEC(m->model, vec, CALL);
#undef CALL
  return 0;
}

long long emu_topk_chunk_rows(long long Q, long long n) { return topk_chunk_rows(Q, n); }

}  // extern "C"
