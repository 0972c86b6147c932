// tests/emu/emu_conve_train.cpp — TEST INFRASTRUCTURE.  Runs ConvE's training-mode trunk kernels of
// pykg2vec_b200/csrc/kge_conve_train.cuh (and the tiled GEMM they launch) on the host, CUDA thread by CUDA thread
// (tests/emu/cuda_runtime.h), with the launch sequence and geometry of kge_conve_train_fwd / _bwd in kge_proj.cu
// (tests/test_emu_conve_train.py).  Built with -DCONVE_TRAIN_RACE_MAIN it is the ThreadSanitizer race check of the
// kernels.  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include <cstdio>
#include <random>

#include "kge_conve_train.cuh"

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

static ConveTrain args(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                       const float* n0, const float* n1, const float* n2, float* ws) {
  ConveTrain a{};
  a.ent = p->ent; a.rel = p->rel; a.e = e; a.r = r;
  a.k = p->hidden_size; a.h1 = p->hidden_size_1; a.h2 = a.k / a.h1; a.Q = Q; a.B = B;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias; a.conv_w = p->conv_weight; a.conv_b = p->conv_bias;
  a.bn1_w = p->bn1_weight; a.bn1_b = p->bn1_bias; a.bn2_w = p->bn2_weight; a.bn2_b = p->bn2_bias;
  a.noise0 = n0; a.noise1 = n1; a.noise2 = n2;
  const ConveTrainLayout L = conve_train_layout(Q, B, a.k, a.h1);
  a.img = ws + L.img; a.z1 = ws + L.z1; a.feat = ws + L.feat; a.hpre = ws + L.hpre;
  a.st0 = ws + L.st0; a.st1 = ws + L.st1; a.st2 = ws + L.st2; a.part0 = ws + L.part0; a.part1 = ws + L.part1;
  a.red0 = ws + L.red0; a.red1 = ws + L.red1; a.dz = ws + L.dz; a.dimg = ws + L.dimg; a.pw = ws + L.pw;
  a.pb = ws + L.pb;
  return a;
}

extern "C" {

int64_t emu_conve_train_workspace_floats(const kge_conve_train_t* p, int64_t Q, int64_t B) {
  return conve_train_layout(Q, B, p->hidden_size, p->hidden_size_1).total;
}

void emu_conve_train_fwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                         const float* n0, const float* n1, const float* n2, float* x, float* ws) {
  const ConveTrain a = args(p, e, r, Q, B, n0, n1, n2, ws);
  const int k = a.k, plane = (2 * a.h2 - 2) * (a.h1 - 2);
  const long long F = conve_feat_width(a.h2, a.h1);
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_gather_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part0, Q, B, 1, (float)(2 * k), p->bn0_eps, p->bn0_momentum, a.st0, p->bn0_mean,
                             p->bn0_var);
  });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_conv_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part1, Q, B, CONVE_CH, (float)plane, p->bn1_eps, p->bn1_momentum, a.st1, p->bn1_mean,
                             p->bn1_var);
  });
  cuda_emu::launch(dim3(proj_tiles(Q * F, 256)), dim3(256), [&] { conve_tr_feat_kernel(a, F, plane); });
  float* partial = ws + conve_train_layout(Q, B, k, a.h1).partial;
  run_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, F, k, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * k, 256)), dim3(256), [&] {
    conve_tr_fc_combine_kernel(partial, conve_fc_slices(F), Q * k, k, p->fc_bias, n2, a.hpre);
  });
  cuda_emu::launch(dim3(proj_tiles(k, 256)), dim3(256),
                   [&] { conve_tr_bn2_kernel(a, p->bn2_eps, p->bn2_momentum, p->bn2_mean, p->bn2_var, x); });
}

void emu_conve_train_bwd(const kge_conve_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                         const float* n0, const float* n1, const float* n2, const float* gx, const float* x,
                         float* const* grads, float* ws) {
  const ConveTrain a = args(p, e, r, Q, B, n0, n1, n2, ws);
  const int k = a.k;
  const long long F = conve_feat_width(a.h2, a.h1);
  float* dh = ws + conve_train_layout(Q, B, k, a.h1).dh;
  cuda_emu::launch(dim3(proj_tiles(k, 256)), dim3(256),
                   [&] { conve_tr_bn2_bwd_kernel(a, gx, x, dh, grads[10], grads[11], grads[9]); });
  run_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(dh, a.feat, Q, F, k, grads[8]));
  run_gemm<EPI_STORE>(conve_plan_grad_feat(dh, p->fc_weight, Q, F, k, a.dz));
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_bn1_bwd_part_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256),
                   [&] { conve_tr_reduce_kernel(a.part1, Q, B, CONVE_CH, a.red1, grads[6], grads[7]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_conv_bwd_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(CONVE_TAPS, 256)), dim3(256),
                   [&] { conve_tr_colsum_kernel(a.pw, Q, CONVE_TAPS, grads[4]); });
  cuda_emu::launch(dim3(1), dim3(256), [&] { conve_tr_colsum_kernel(a.pb, Q, CONVE_CH, grads[5]); });
  cuda_emu::launch(dim3(1), dim3(256), [&] { conve_tr_reduce_kernel(a.part0, Q, B, 1, a.red0, grads[2], grads[3]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_bn0_bwd_kernel(a, grads[0], grads[1]); });
}

}  // extern "C"

#ifdef CONVE_TRAIN_RACE_MAIN
// ThreadSanitizer build: the three CTA-per-query kernels pass the image, z1 and dz through shared memory and
// __syncthreads, the CTA sums through a shared array; two groups, queries sharing an entity and a relation
int main(int argc, char**) {
  if (argc > 1) return 64;   // "probe": only the sanitizer runtime starts
  const int k = 20, h1 = 4, N = 5, R = 3, B = 3, Q = 6, F = 32 * 8 * 2;
  std::mt19937 gen(7);
  std::normal_distribution<float> nd(0.f, 0.5f);
  auto rnd = [&](size_t n) { std::vector<float> v(n); for (auto& y : v) y = nd(gen); return v; };
  auto ent = rnd(N * k), rel = rnd(2 * R * k), cw = rnd(288), cb = rnd(32), fw = rnd((size_t)k * F), fb = rnd(k);
  auto gx = rnd(Q * k), n0 = rnd(Q * 2 * k), n1 = rnd(Q * 32), n2 = rnd(Q * k);
  std::vector<float> w0{1.1f}, b0{0.1f}, w1(32, 0.9f), b1(32, 0.05f), w2(k, 1.2f), b2(k, -0.1f);
  std::vector<float> rm0(1, 0.f), rv0(1, 1.f), rm1(32, 0.f), rv1(32, 1.f), rm2(k, 0.f), rv2(k, 1.f);
  kge_conve_train_t p{k, h1, 1e-5f, 1e-5f, 1e-5f, 0.1f, 0.1f, 0.1f, ent.data(), rel.data(), w0.data(), b0.data(),
                      cw.data(), cb.data(), w1.data(), b1.data(), fw.data(), fb.data(), w2.data(), b2.data(),
                      rm0.data(), rv0.data(), rm1.data(), rv1.data(), rm2.data(), rv2.data()};
  std::vector<int64_t> e = {4, 1, 4, 0, 4, 2}, r = {2, 0, 2, 5, 3, 2};
  std::vector<float> ws(emu_conve_train_workspace_floats(&p, Q, B)), x(Q * k);
  std::vector<std::vector<float>> g = {std::vector<float>(N * k), std::vector<float>(2 * R * k), std::vector<float>(1),
                                       std::vector<float>(1), std::vector<float>(288), std::vector<float>(32),
                                       std::vector<float>(32), std::vector<float>(32), std::vector<float>(k * F),
                                       std::vector<float>(k), std::vector<float>(k), std::vector<float>(k)};
  float* gp[12];
  for (int i = 0; i < 12; ++i) gp[i] = g[i].data();
  emu_conve_train_fwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), x.data(), ws.data());
  emu_conve_train_bwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), gx.data(), x.data(), gp,
                      ws.data());
  printf("%g %g\n", x[0], g[0][0]);
  return 0;
}
#endif
