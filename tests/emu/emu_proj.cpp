// tests/emu/emu_proj.cpp — TEST INFRASTRUCTURE.  Runs the projection-tail kernels of
// pykg2vec_b200/csrc/kge_proj.cuh on the host, CUDA thread by CUDA thread (tests/emu/cuda_runtime.h),
// with the SAME launch plans the C-ABI launchers use, so the tiling, strides, split-K ranges,
// padding, shuffles and atomics are checked against the oracle without a GPU
// (tests/test_emu_proj.py).  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include "kge_conve.cuh"

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

template <int EPI>
static void run_gemm(const ProjLaunch& L) {
  const dim3 grid(L.gx, L.gy, L.gz);
  switch (L.tile) {
    case PROJ_TILE_128x128: cuda_emu::launch(grid, dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 8, 8>(L.g); }); break;
    case PROJ_TILE_64x128: cuda_emu::launch(grid, dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 4, 8>(L.g); }); break;
    default: cuda_emu::launch(grid, dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 4, 4>(L.g); }); break;
  }
}

extern "C" {

int emu_proj_tail_fwd(const float* x, const float* ent, const float* bias, int64_t B, int64_t N, int32_t k,
                      float* preds, int32_t tile) {
  run_gemm<EPI_STORE>(proj_plan_fwd(x, ent, bias, B, N, k, preds, tile));
  return 0;
}

int emu_proj_tail_bwd(const float* grad_preds, const float* preds, const float* x, const float* ent, int64_t B,
                      int64_t N, int32_t k, float* grad_x, float* grad_ent, float* grad_bias, int32_t target_ctas) {
  if (grad_x) run_gemm<EPI_ATOMIC>(proj_plan_grad_x(grad_preds, preds, ent, B, N, k, grad_x, target_ctas));
  if (grad_ent) run_gemm<EPI_ATOMIC>(proj_plan_grad_ent(grad_preds, preds, x, B, N, k, grad_ent));
  if (grad_bias)
    cuda_emu::launch(dim3(proj_tiles(N, 256)), dim3(256),
                     [&] { proj_colsum_kernel(grad_preds, preds, (int)B, N, grad_bias); });
  return 0;
}

int emu_proj_bce(const float* preds, const float* labels, int64_t B, int64_t N, float label_scale,
                 float label_shift, float grad_scale, float* loss_out, float* grad_preds, int32_t sms) {
  const long long n = (long long)B * N;
  loss_out[0] = 0.f;
  cuda_emu::launch(dim3(proj_bce_blocks(n, sms)), dim3(256), [&] {
    proj_bce_kernel(preds, labels, n, label_scale, label_shift, proj_bce_grad_factor(grad_scale, B, N),
                    proj_bce_inv_count(B, N), loss_out, grad_preds);
  });
  return 0;
}

int emu_proj_rank(const float* x, const float* ent, const float* bias, int64_t Q, int64_t N, int32_t k,
                  const int64_t* tgt, const int64_t* filt_ptr, const int64_t* filt_idx, int64_t filt_nnz,
                  int32_t direction, int32_t* counts, float* thr, int32_t tile) {
  cuda_emu::launch(dim3(proj_tiles(Q, 128)), dim3(128),
                   [&] { proj_target_kernel(x, ent, bias, tgt, (int)Q, k, thr); });
  run_gemm<EPI_COUNT>(proj_plan_count(x, ent, bias, Q, N, k, thr, counts, direction, tile));
  if (filt_ptr && filt_idx && filt_nnz > 0)
    cuda_emu::launch(dim3((unsigned)Q), dim3(128), [&] {
      proj_filter_kernel(x, ent, bias, tgt, filt_ptr, filt_idx, k, thr, counts, 2 * direction);
    });
  return 0;
}

int emu_proj_labels(const int64_t* rows, const int64_t* ptr, const int64_t* idx, int64_t B, int64_t N,
                    float* labels) {
  memset(labels, 0, sizeof(float) * (size_t)B * (size_t)N);
  cuda_emu::launch(dim3((unsigned)B), dim3(128), [&] { proj_labels_kernel(rows, ptr, idx, N, labels); });
  return 0;
}

int emu_conve_trunk_fwd(const kge_conve_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x,
                        float* feat) {
  const int k = p->hidden_size, h1 = p->hidden_size_1, h2 = k / h1;
  ConveFeat f{};
  f.ent = p->ent; f.rel = p->rel; f.e = e; f.r = r; f.k = k; f.h2 = h2; f.h1 = h1;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.conv_w = p->conv_weight; f.conv_b = p->conv_bias;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  f.feat = feat;
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_THREADS), [&] { conve_feature_kernel(f); });
  const long long F = conve_feat_width(h2, h1);
  float* partial = feat + Q * F;   // the caller sizes feat as the C-ABI workspace: [Q,F] + [slices,Q,k]
  run_gemm<EPI_STORE>(conve_plan_fc(feat, p->fc_weight, Q, F, k, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * k, 256)), dim3(256), [&] {
    conve_fc_combine_kernel(partial, conve_fc_slices(F), Q * k, k, p->fc_bias, x);
  });
  return 0;
}

}  // extern "C"
