// tests/emu/emu_hyper_train.cpp — TEST INFRASTRUCTURE.  Runs HypER's training-mode trunk kernels of
// pykg2vec_b200/csrc/kge_hyper_train.cuh (and the tiled GEMM and kge_conve_train.cuh kernels they launch) on the host,
// CUDA thread by CUDA thread (tests/emu/cuda_runtime.h), with the launch sequence and geometry of kge_hyper_train_fwd /
// _bwd in kge_proj.cu (tests/test_emu_hyper_train.py).  Built with -DHYPER_TRAIN_RACE_MAIN it is the ThreadSanitizer
// race check of the kernels.  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include <cstdio>
#include <random>

#include "kge_hyper_train.cuh"

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
  cuda_emu::launch(dim3(L.gx, L.gy, L.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI, 4, 4>(L.g); });
}

static HyperTrain args(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                       const float* n0, const float* n1, const float* n2, float* ws) {
  HyperTrain a{};
  a.ent = p->ent; a.e = e; a.r = r;
  a.de = p->ent_hidden_size; a.dr = p->rel_hidden_size; a.Q = Q; a.B = B;
  a.ent_pad = p->ent_padding_idx; a.rel_pad = p->rel_padding_idx;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias; a.bn1_w = p->bn1_weight; a.bn1_b = p->bn1_bias;
  a.bn2_w = p->bn2_weight; a.bn2_b = p->bn2_bias;
  a.noise0 = n0; a.noise1 = n1; a.noise2 = n2;
  const HyperTrainLayout L = hyper_train_layout(Q, B, a.de, a.dr);
  a.relr = ws + L.relr; a.filt = ws + L.filt; a.img = ws + L.img; a.z1 = ws + L.z1; a.feat = ws + L.feat;
  a.hpre = ws + L.hpre; a.st0 = ws + L.st0; a.st1 = ws + L.st1; a.st2 = ws + L.st2; a.part0 = ws + L.part0;
  a.part1 = ws + L.part1; a.red0 = ws + L.red0; a.red1 = ws + L.red1; a.dh = ws + L.dh; a.dz = ws + L.dz;
  a.dimg = ws + L.dimg; a.dw = ws + L.dw; a.drel = ws + L.drel;
  return a;
}

extern "C" {

int64_t emu_hyper_train_workspace_floats(const kge_hyper_train_t* p, int64_t Q, int64_t B) {
  return hyper_train_layout(Q, B, p->ent_hidden_size, p->rel_hidden_size).total;
}

void emu_hyper_train_fwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                         const float* n0, const float* n1, const float* n2, float* x, float* ws) {
  const HyperTrain a = args(p, e, r, Q, B, n0, n1, n2, ws);
  const int de = a.de, dr = a.dr, Wo = de - HYPER_FW + 1;
  const long long F = hyper_feat_width(de);
  cuda_emu::launch(dim3(proj_tiles(Q * dr, 256)), dim3(256),
                   [&] { tucker_gather_rows_kernel(p->rel, r, Q, dr, a.relr); });
  run_gemm<EPI_STORE>(hyper_plan_filters(a.relr, p->fc1_weight, p->fc1_bias, Q, dr, a.filt));
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { hyper_tr_gather_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part0, Q, B, 1, (float)de, p->bn0_eps, p->bn0_momentum, a.st0, p->bn0_mean,
                             p->bn0_var);
  });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { hyper_tr_conv_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part1, Q, B, HYPER_CH, (float)Wo, p->bn1_eps, p->bn1_momentum, a.st1, p->bn1_mean,
                             p->bn1_var);
  });
  cuda_emu::launch(dim3(proj_tiles(Q * F, 256)), dim3(256), [&] { hyper_tr_feat_kernel(a, F, Wo); });
  float* partial = ws + hyper_train_layout(Q, B, de, dr).partial;
  run_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, F, de, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * de, 256)), dim3(256), [&] {
    conve_tr_fc_combine_kernel(partial, conve_fc_slices(F), Q * de, de, p->fc_bias, n2, a.hpre);
  });
  cuda_emu::launch(dim3(proj_tiles(de, 256)), dim3(256), [&] {
    conve_tr_bn2_kernel(hyper_tr_bn2_view(a), p->bn2_eps, p->bn2_momentum, p->bn2_mean, p->bn2_var, x);
  });
}

void emu_hyper_train_bwd(const kge_hyper_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                         const float* n0, const float* n1, const float* n2, const float* gx, const float* x,
                         float* const* grads, float* ws) {
  const HyperTrain a = args(p, e, r, Q, B, n0, n1, n2, ws);
  const int de = a.de, dr = a.dr;
  const long long F = hyper_feat_width(de);
  cuda_emu::launch(dim3(proj_tiles(de, 256)), dim3(256),
                   [&] { conve_tr_bn2_bwd_kernel(hyper_tr_bn2_view(a), gx, x, a.dh, grads[8], grads[9], grads[7]); });
  run_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.dh, a.feat, Q, F, de, grads[6]));
  run_gemm<EPI_STORE>(conve_plan_grad_feat(a.dh, p->fc_weight, Q, F, de, a.dz));
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { hyper_tr_bn1_bwd_part_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256),
                   [&] { conve_tr_reduce_kernel(a.part1, Q, B, HYPER_CH, a.red1, grads[4], grads[5]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { hyper_tr_conv_bwd_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256), [&] { conve_tr_reduce_kernel(a.part0, Q, B, 1, a.red0, grads[2], grads[3]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { hyper_tr_bn0_bwd_kernel(a, grads[0]); });
  run_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.dw, a.relr, Q, dr, HYPER_FILT, grads[10]));
  cuda_emu::launch(dim3(proj_tiles(HYPER_FILT, 256)), dim3(256),
                   [&] { conve_tr_colsum_kernel(a.dw, Q, HYPER_FILT, grads[11]); });
  run_gemm<EPI_STORE>(conve_plan_grad_feat(a.dw, p->fc1_weight, Q, dr, HYPER_FILT, a.drel));
  cuda_emu::launch(dim3(proj_tiles(Q * dr, 256)), dim3(256),
                   [&] { hyper_tr_scatter_rel_kernel(a.drel, r, Q, dr, a.rel_pad, grads[1]); });
}

}  // extern "C"

#ifdef HYPER_TRAIN_RACE_MAIN
// ThreadSanitizer build: the CTA-per-query kernels pass the bn0 output, the filters, z1 and dz through shared memory,
// global memory and __syncthreads, the CTA sums through a shared array; two groups, queries sharing an entity and a
// relation, the padding id 0 among them
int main(int argc, char**) {
  if (argc > 1) return 64;   // "probe": only the sanitizer runtime starts
  const int de = 20, dr = 6, N = 5, R = 3, B = 3, Q = 6, F = 32 * 12;
  std::mt19937 gen(7);
  std::normal_distribution<float> nd(0.f, 0.5f);
  auto rnd = [&](size_t n) { std::vector<float> v(n); for (auto& y : v) y = nd(gen); return v; };
  auto ent = rnd(N * de), rel = rnd(R * dr), fw = rnd((size_t)de * F), fb = rnd(de), f1w = rnd(288 * dr), f1b = rnd(288);
  auto gx = rnd(Q * de), n0 = rnd(Q * de), n1 = rnd(Q * 32), n2 = rnd(Q * de);
  std::vector<float> w0{1.1f}, b0{0.1f}, w1(32, 0.9f), b1(32, 0.05f), w2(de, 1.2f), b2(de, -0.1f);
  std::vector<float> rm0(1, 0.f), rv0(1, 1.f), rm1(32, 0.f), rv1(32, 1.f), rm2(de, 0.f), rv2(de, 1.f);
  kge_hyper_train_t p{de, dr, 0, 0, 1e-5f, 1e-5f, 1e-5f, 0.1f, 0.1f, 0.1f, ent.data(), rel.data(), w0.data(),
                      b0.data(), w1.data(), b1.data(), fw.data(), fb.data(), w2.data(), b2.data(), f1w.data(),
                      f1b.data(), rm0.data(), rv0.data(), rm1.data(), rv1.data(), rm2.data(), rv2.data()};
  std::vector<int64_t> e = {4, 1, 4, 0, 4, 2}, r = {2, 0, 2, 1, 0, 2};
  std::vector<float> ws(emu_hyper_train_workspace_floats(&p, Q, B)), x(Q * de);
  std::vector<std::vector<float>> g = {std::vector<float>(N * de), std::vector<float>(R * dr), std::vector<float>(1),
                                       std::vector<float>(1), std::vector<float>(32), std::vector<float>(32),
                                       std::vector<float>(de * F), std::vector<float>(de), std::vector<float>(de),
                                       std::vector<float>(de), std::vector<float>(288 * dr), std::vector<float>(288)};
  float* gp[12];
  for (int i = 0; i < 12; ++i) gp[i] = g[i].data();
  emu_hyper_train_fwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), x.data(), ws.data());
  emu_hyper_train_bwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), gx.data(), x.data(), gp,
                      ws.data());
  printf("%g %g\n", x[0], g[0][de]);
  return 0;
}
#endif
