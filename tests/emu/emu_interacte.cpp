// tests/emu/emu_interacte.cpp — TEST INFRASTRUCTURE.  Runs InteractE's inference-trunk kernels of
// pykg2vec_b200/csrc/kge_interacte.cuh (feature kernel, sliced Linear GEMM, combine) on the host, CUDA thread by
// CUDA thread (tests/emu/cuda_runtime.h), with the SAME layout and launch plans the C-ABI launcher
// kge_interacte_trunk_fwd uses (tests/test_emu_interacte.py).  Not a product path: nothing in pykg2vec_b200/
// can reach it.
#include "kge_interacte.cuh"

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
}  // namespace kge

using namespace kge;

extern "C" {

// workspace floats the caller must provide (= kge_interacte_trunk_workspace_bytes / 4)
int64_t emu_interacte_workspace_floats(const kge_interacte_t* p, int64_t Q) {
  return interacte_layout(Q, p->feature_permutation, p->num_filters, 2 * p->reshape_width, p->reshape_height).total;
}

// shared-memory bytes of the feature kernel (the launcher's dynamic allocation)
int64_t emu_interacte_smem_bytes(const kge_interacte_t* p) {
  return interacte_smem(p->feature_permutation, p->num_filters, p->kernel_size, 2 * p->reshape_width,
                        p->reshape_height).total * (int64_t)sizeof(float);
}

int emu_interacte_trunk_fwd(const kge_interacte_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                            float* ws) {
  const int P = p->feature_permutation, F = p->num_filters, H = 2 * p->reshape_width, W = p->reshape_height;
  const int k = p->reshape_width * p->reshape_height;
  if (emu_interacte_smem_bytes(p) > INTERACTE_SMEM_MAX) return KGE_ENOTSUP;
  const InteracteLayout lay = interacte_layout(Q, P, F, H, W);
  InteracteFeat f{};
  f.ent = p->ent; f.rel = p->rel; f.perm = p->perm; f.e = e; f.r = r;
  f.P = P; f.F = F; f.ks = p->kernel_size; f.H = H; f.W = W;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.conv_filt = p->conv_filt;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  f.feat = ws + lay.feat;
  cuda_emu::launch(dim3((unsigned)Q), dim3(INTERACTE_THREADS), [&] { interacte_feature_kernel(f); });
  const long long Fw = interacte_feat_width(P, F, H, W);
  float* partial = ws + lay.partial;
  const ProjLaunch L = conve_plan_fc(f.feat, p->fc_weight, Q, Fw, k, partial);   // the 64x64 tile, as launched
  cuda_emu::launch(dim3(L.gx, L.gy, L.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI_STORE, 4, 4>(L.g); });
  cuda_emu::launch(dim3(proj_tiles(Q * k, 256)), dim3(256), [&] {
    hyper_fc_combine_kernel(partial, conve_fc_slices(Fw), Q * k, k, p->fc_bias, p->bn2_weight, p->bn2_bias,
                            p->bn2_mean, p->bn2_var, p->bn2_eps, x);
  });
  return 0;
}

}  // extern "C"
