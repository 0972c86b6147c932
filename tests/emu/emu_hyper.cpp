// tests/emu/emu_hyper.cpp — TEST INFRASTRUCTURE.  Runs HypER's inference-trunk kernels of
// pykg2vec_b200/csrc/kge_hyper.cuh (filter GEMM, feature kernel, sliced Linear GEMM, combine) on the host,
// CUDA thread by CUDA thread (tests/emu/cuda_runtime.h), with the SAME layout and launch plans the C-ABI
// launcher kge_hyper_trunk_fwd uses (tests/test_emu_hyper.py).  Not a product path: nothing in
// pykg2vec_b200/ can reach it.
#include "kge_hyper.cuh"

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

static void run_store_gemm(const ProjLaunch& L) {   // both plans use the 64x64 tile, as the launcher does
  cuda_emu::launch(dim3(L.gx, L.gy, L.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI_STORE, 4, 4>(L.g); });
}

extern "C" {

// workspace floats the caller must provide (= kge_hyper_trunk_workspace_bytes / 4)
int64_t emu_hyper_workspace_floats(int64_t R, int64_t Q, int32_t de) { return hyper_layout(R, Q, de).total; }

// offsets (floats) of the filter table and the features inside the workspace
void emu_hyper_layout(int64_t R, int64_t Q, int32_t de, int64_t* filt, int64_t* feat) {
  const HyperLayout L = hyper_layout(R, Q, de);
  *filt = L.filt;
  *feat = L.feat;
}

int emu_hyper_trunk_fwd(const kge_hyper_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x, float* ws) {
  const int de = p->ent_hidden_size;
  const HyperLayout lay = hyper_layout(p->num_rel, Q, de);
  run_store_gemm(hyper_plan_filters(p->rel, p->fc1_weight, p->fc1_bias, p->num_rel, p->rel_hidden_size, ws + lay.filt));
  HyperFeat f{};
  f.ent = p->ent; f.filt = ws + lay.filt; f.e = e; f.r = r; f.de = de;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  f.feat = ws + lay.feat;
  cuda_emu::launch(dim3((unsigned)Q), dim3(HYPER_THREADS), [&] { hyper_feature_kernel(f); });
  const long long F = hyper_feat_width(de);
  float* partial = ws + lay.partial;
  run_store_gemm(conve_plan_fc(f.feat, p->fc_weight, Q, F, de, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * de, 256)), dim3(256), [&] {
    hyper_fc_combine_kernel(partial, conve_fc_slices(F), Q * de, de, p->fc_bias, p->bn2_weight, p->bn2_bias,
                            p->bn2_mean, p->bn2_var, p->bn2_eps, x);
  });
  return 0;
}

}  // extern "C"
