// tests/emu/emu_interacte_train.cpp — TEST INFRASTRUCTURE.  Runs InteractE's training-mode trunk kernels of
// pykg2vec_b200/csrc/kge_interacte_train.cuh (and the tiled GEMM and kge_conve_train.cuh kernels they launch) on the
// host, CUDA thread by CUDA thread (tests/emu/cuda_runtime.h), with the launch sequence and geometry of
// kge_interacte_train_fwd / _bwd in kge_proj.cu (tests/test_emu_interacte_train.py).  Built with
// -DINTERACTE_TRAIN_RACE_MAIN it is the ThreadSanitizer race check of the kernels.  Not a product path: nothing in
// pykg2vec_b200/ can reach it.
#include <cstdio>
#include <random>

#include "kge_interacte_train.cuh"

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

static InteracteTrainLayout layout(const kge_interacte_train_t* p, int64_t Q, int64_t B) {
  return interacte_train_layout(Q, B, p->feature_permutation, p->num_filters, p->kernel_size, 2 * p->reshape_width,
                                p->reshape_height);
}

static InteracteTrain args(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                           const float* n0, const float* n1, const float* n2, float* ws) {
  InteracteTrain a{};
  a.ent = p->ent; a.rel = p->rel; a.perm = p->perm; a.e = e; a.r = r;
  a.P = p->feature_permutation; a.F = p->num_filters; a.ks = p->kernel_size;
  a.H = 2 * p->reshape_width; a.W = p->reshape_height; a.Q = Q; a.B = B;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias; a.filt = p->conv_filt; a.bn1_w = p->bn1_weight;
  a.bn1_b = p->bn1_bias; a.bn2_w = p->bn2_weight; a.bn2_b = p->bn2_bias;
  a.noise0 = n0; a.noise1 = n1; a.noise2 = n2;
  const InteracteTrainLayout L = layout(p, Q, B);
  a.img = ws + L.img; a.z1 = ws + L.z1; a.feat = ws + L.feat; a.hpre = ws + L.hpre; a.st0 = ws + L.st0;
  a.st1 = ws + L.st1; a.st2 = ws + L.st2; a.part0 = ws + L.part0; a.part1 = ws + L.part1; a.red0 = ws + L.red0;
  a.red1 = ws + L.red1; a.dh = ws + L.dh; a.dimg = ws + L.dimg; a.pw = ws + L.pw;
  return a;
}

extern "C" {

int64_t emu_interacte_train_workspace_floats(const kge_interacte_train_t* p, int64_t Q, int64_t B) {
  return layout(p, Q, B).total;
}

void emu_interacte_train_fwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                             const float* n0, const float* n1, const float* n2, float* x, float* ws) {
  const InteracteTrain a = args(p, e, r, Q, B, n0, n1, n2, ws);
  const int P = a.P, F = a.F, HW = a.H * a.W, k = HW / 2, C1 = P * F;
  const long long Fw = (long long)C1 * HW;
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { interacte_tr_gather_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(P, 256)), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part0, Q, B, P, (float)HW, p->bn0_eps, p->bn0_momentum, a.st0, p->bn0_mean, p->bn0_var);
  });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { interacte_tr_conv_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(C1, 256)), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part1, Q, B, C1, (float)HW, p->bn1_eps, p->bn1_momentum, a.st1, p->bn1_mean,
                             p->bn1_var);
  });
  cuda_emu::launch(dim3(proj_tiles(Q * Fw, 256)), dim3(256), [&] { interacte_tr_feat_kernel(a, Fw, HW); });
  float* partial = ws + layout(p, Q, B).partial;
  run_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, Fw, k, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * k, 256)), dim3(256), [&] {
    conve_tr_fc_combine_kernel(partial, conve_fc_slices(Fw), Q * k, k, p->fc_bias, n2, a.hpre);
  });
  cuda_emu::launch(dim3(proj_tiles(k, 256)), dim3(256), [&] {
    conve_tr_bn2_kernel(interacte_tr_bn2_view(a), p->bn2_eps, p->bn2_momentum, p->bn2_mean, p->bn2_var, x);
  });
}

void emu_interacte_train_bwd(const kge_interacte_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                             const float* n0, const float* n1, const float* n2, const float* gx, const float* x,
                             float* const* grads, float* ws) {
  const InteracteTrain a = args(p, e, r, Q, B, n0, n1, n2, ws);
  const int P = a.P, F = a.F, HW = a.H * a.W, k = HW / 2, C1 = P * F, taps = a.ks * a.ks;
  const long long Fw = (long long)C1 * HW;
  cuda_emu::launch(dim3(proj_tiles(k, 256)), dim3(256), [&] {
    conve_tr_bn2_bwd_kernel(interacte_tr_bn2_view(a), gx, x, a.dh, grads[9], grads[10], grads[8]);
  });
  run_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.dh, a.feat, Q, Fw, k, grads[7]));
  run_gemm<EPI_STORE>(conve_plan_grad_feat(a.dh, p->fc_weight, Q, Fw, k, a.feat));
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { interacte_tr_bn1_bwd_part_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(C1, 256)), dim3(256),
                   [&] { conve_tr_reduce_kernel(a.part1, Q, B, C1, a.red1, grads[5], grads[6]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { interacte_tr_conv_bwd_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(F * taps, 256)), dim3(256),
                   [&] { conve_tr_colsum_kernel(a.pw, Q, F * taps, grads[4]); });
  cuda_emu::launch(dim3(proj_tiles(P, 256)), dim3(256),
                   [&] { conve_tr_reduce_kernel(a.part0, Q, B, P, a.red0, grads[2], grads[3]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS),
                   [&] { interacte_tr_bn0_bwd_kernel(a, grads[0], grads[1]); });
}

}  // extern "C"

#ifdef INTERACTE_TRAIN_RACE_MAIN
// ThreadSanitizer build: the CTA-per-query kernels pass the padded bn0 outputs, the filter bank, z1, dz1, dimg and the
// inverse permutations through shared memory, global memory and __syncthreads, the CTA sums through a shared array;
// two groups of P = 2 images, queries sharing an entity and a relation
int main(int argc, char**) {
  if (argc > 1) return 64;   // "probe": only the sanitizer runtime starts
  const int P = 2, F = 3, ks = 3, rh = 3, rw = 2, k = rh * rw, HW = 2 * k, N = 5, R = 3, B = 3, Q = 6;
  const int C1 = P * F, Fw = C1 * HW;
  std::mt19937 gen(7);
  std::normal_distribution<float> nd(0.f, 0.5f);
  auto rnd = [&](size_t n) { std::vector<float> v(n); for (auto& y : v) y = nd(gen); return v; };
  auto ent = rnd(N * k), rel = rnd(R * k), filt = rnd(F * ks * ks), fw = rnd((size_t)k * Fw), fb = rnd(k);
  auto gx = rnd(Q * k), n0 = rnd(Q * P * HW), n1 = rnd(Q * C1), n2 = rnd(Q * k);
  std::vector<float> w0(P, 1.1f), b0(P, 0.1f), w1(C1, 0.9f), b1(C1, 0.05f), w2(k, 1.2f), b2(k, -0.1f);
  std::vector<float> rm0(P, 0.f), rv0(P, 1.f), rm1(C1, 0.f), rv1(C1, 1.f), rm2(k, 0.f), rv2(k, 1.f);
  std::vector<int64_t> perm(P * HW);
  for (int p = 0; p < P; ++p)
    for (int i = 0; i < HW; ++i) perm[p * HW + i] = (i * (2 * p + 5) + p) % HW;   // 5 and 7 are prime to 12
  kge_interacte_train_t p{P, F, ks, rh, rw, 1e-5f, 1e-5f, 1e-5f, 0.1f, 0.1f, 0.1f, perm.data(), ent.data(),
                          rel.data(), w0.data(), b0.data(), filt.data(), w1.data(), b1.data(), fw.data(), fb.data(),
                          w2.data(), b2.data(), rm0.data(), rv0.data(), rm1.data(), rv1.data(), rm2.data(), rv2.data()};
  std::vector<int64_t> e = {4, 1, 4, 0, 4, 2}, r = {2, 0, 2, 1, 0, 2};
  std::vector<float> ws(emu_interacte_train_workspace_floats(&p, Q, B)), x(Q * k);
  std::vector<std::vector<float>> g = {std::vector<float>(N * k), std::vector<float>(R * k), std::vector<float>(P),
                                       std::vector<float>(P), std::vector<float>(F * ks * ks), std::vector<float>(C1),
                                       std::vector<float>(C1), std::vector<float>((size_t)k * Fw),
                                       std::vector<float>(k), std::vector<float>(k), std::vector<float>(k)};
  float* gp[11];
  for (int i = 0; i < 11; ++i) gp[i] = g[i].data();
  emu_interacte_train_fwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), x.data(), ws.data());
  emu_interacte_train_bwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), gx.data(), x.data(), gp,
                          ws.data());
  printf("%g %g\n", x[0], g[0][k]);
  return 0;
}
#endif
