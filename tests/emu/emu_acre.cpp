// tests/emu/emu_acre.cpp — TEST INFRASTRUCTURE.  Runs AcrE's inference-trunk kernels of
// pykg2vec_b200/csrc/kge_acre.cuh (serial feature kernel, or gate-input kernel + W_gate_e GEMM + bn1/ReLU; then
// the sliced Linear GEMM and the combine) on the host, CUDA thread by CUDA thread (tests/emu/cuda_runtime.h),
// with the SAME layout and launch plans the C-ABI launcher kge_acre_trunk_fwd uses (tests/test_emu_acre.py).
// Not a product path: nothing in pykg2vec_b200/ can reach it.
#include "kge_acre.cuh"

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

// workspace floats the caller must provide (= kge_acre_trunk_workspace_bytes / 4)
int64_t emu_acre_workspace_floats(const kge_acre_t* p, int64_t Q) {
  return acre_layout(Q, p->in_channels, p->way == 1).total;
}

// {gate, feat, partial} offsets of the workspace, in floats
void emu_acre_layout(const kge_acre_t* p, int64_t Q, int64_t* out) {
  const AcreLayout L = acre_layout(Q, p->in_channels, p->way == 1);
  out[0] = L.gate; out[1] = L.feat; out[2] = L.partial;
}

// dynamic shared-memory bytes of the way's feature kernel (the launcher's allocation)
int64_t emu_acre_smem_bytes(const kge_acre_t* p) {
  return (p->way == 0 ? acre_serial_smem(p->in_channels).total : acre_gate_smem(p->in_channels)) *
         (int64_t)sizeof(float);
}

int emu_acre_trunk_fwd(const kge_acre_t* p, const int64_t* e, const int64_t* r, int64_t Q, float* x, float* ws) {
  const int C = p->in_channels;
  const bool par = p->way == 1;
  if (emu_acre_smem_bytes(p) > ACRE_SMEM_MAX) return KGE_ENOTSUP;
  const AcreLayout lay = acre_layout(Q, C, par);
  AcreFeat f{};
  f.ent = p->ent; f.rel = p->rel; f.e = e; f.r = r; f.C = C;
  f.dil[0] = p->first_atrous; f.dil[1] = p->second_atrous; f.dil[2] = p->third_atrous;
  f.bn0_w = p->bn0_weight; f.bn0_b = p->bn0_bias; f.bn0_mean = p->bn0_mean; f.bn0_var = p->bn0_var;
  f.bn0_eps = p->bn0_eps;
  f.conv_w[0] = p->conv1_weight; f.conv_w[1] = p->conv2_weight; f.conv_w[2] = p->conv3_weight;
  f.conv_b[0] = p->conv1_bias; f.conv_b[1] = p->conv2_bias; f.conv_b[2] = p->conv3_bias;
  f.bn1_w = p->bn1_weight; f.bn1_b = p->bn1_bias; f.bn1_mean = p->bn1_mean; f.bn1_var = p->bn1_var;
  f.bn1_eps = p->bn1_eps;
  float* feat = ws + lay.feat;
  if (!par) {
    f.out = feat;
    cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_THREADS), [&] { acre_serial_feature_kernel(f); });
  } else {
    f.out = ws + lay.gate;
    cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_GATE_THREADS), [&] { acre_gate_input_kernel(f); });
    const long long rows = Q * C;
    const ProjLaunch G = acre_plan_gate(f.out, p->W_gate_e_weight, p->W_gate_e_bias, rows, feat,
                                        PROJ_TILE_64x64);   // every tile runs the same chain
    cuda_emu::launch(dim3(G.gx, G.gy, G.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI_STORE, 4, 4>(G.g); });
    cuda_emu::launch(dim3(proj_tiles(rows * ACRE_PIX, 256)), dim3(256), [&] {
      acre_bn1_relu_kernel(feat, rows * ACRE_PIX, C, p->bn1_weight, p->bn1_bias, p->bn1_mean, p->bn1_var,
                           p->bn1_eps);
    });
  }
  const long long Fw = acre_feat_width(C);
  float* partial = ws + lay.partial;
  const ProjLaunch L = conve_plan_fc(feat, p->fc_weight, Q, Fw, ACRE_K, partial);   // the 64x64 tile, as launched
  cuda_emu::launch(dim3(L.gx, L.gy, L.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI_STORE, 4, 4>(L.g); });
  cuda_emu::launch(dim3(proj_tiles(Q * ACRE_K, 256)), dim3(256), [&] {
    hyper_fc_combine_kernel(partial, conve_fc_slices(Fw), Q * ACRE_K, ACRE_K, p->fc_bias, p->bn2_weight,
                            p->bn2_bias, p->bn2_mean, p->bn2_var, p->bn2_eps, x);
  });
  return 0;
}

}  // extern "C"
