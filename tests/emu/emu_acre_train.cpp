// tests/emu/emu_acre_train.cpp — TEST INFRASTRUCTURE.  Runs AcrE's training-mode trunk kernels of
// pykg2vec_b200/csrc/kge_acre_train.cuh (and the tiled GEMM and kge_conve_train.cuh kernels they launch) on the host,
// CUDA thread by CUDA thread (tests/emu/cuda_runtime.h), with the launch sequence and geometry of kge_acre_train_fwd /
// _bwd in kge_proj.cu (tests/test_emu_acre_train.py).  Built with -DACRE_TRAIN_RACE_MAIN it is the ThreadSanitizer
// race check of the kernels.  Not a product path: nothing in pykg2vec_b200/ can reach it.
#include <cstdio>
#include <random>

#include "kge_acre_train.cuh"

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

static AcreTrain args(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                      const float* n0, const float* n1, float* ws) {
  AcreTrain a{};
  a.ent = p->ent; a.rel = p->rel; a.e = e; a.r = r;
  a.C = p->in_channels; a.dil[0] = p->first_atrous; a.dil[1] = p->second_atrous; a.dil[2] = p->third_atrous;
  a.par = p->way == 1; a.has_bias = p->conv1_bias != nullptr; a.Q = Q; a.B = B;
  a.bn0_w = p->bn0_weight; a.bn0_b = p->bn0_bias;
  a.conv_w[0] = p->conv1_weight; a.conv_w[1] = p->conv2_weight; a.conv_w[2] = p->conv3_weight;
  a.conv_b[0] = p->conv1_bias; a.conv_b[1] = p->conv2_bias; a.conv_b[2] = p->conv3_bias;
  a.bn1_w = p->bn1_weight; a.bn1_b = p->bn1_bias; a.noise0 = n0; a.noise1 = n1;
  const AcreTrainLayout L = acre_train_layout(Q, B, a.C, a.par);
  a.img = ws + L.img; a.y = ws + L.y; a.feat = ws + L.feat; a.a1 = ws + L.a1; a.a2 = ws + L.a2; a.gate = ws + L.gate;
  a.st0 = ws + L.st0; a.st1 = ws + L.st1; a.part0 = ws + L.part0; a.part1 = ws + L.part1; a.red1 = ws + L.red1;
  a.dimg = ws + L.dimg;
  for (int l = 0; l < 3; ++l) { a.pw[l] = ws + L.pw[l]; a.pb[l] = ws + L.pb[l]; }
  return a;
}

extern "C" {

int64_t emu_acre_train_workspace_floats(const kge_acre_train_t* p, int64_t Q, int64_t B) {
  return acre_train_layout(Q, B, p->in_channels, p->way == 1).total;
}

void emu_acre_train_fwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* n0, const float* n1, const float* n2, float* x, float* ws) {
  const AcreTrain a = args(p, e, r, Q, B, n0, n1, ws);
  const AcreTrainLayout L = acre_train_layout(Q, B, a.C, a.par);
  const ConveTrain cv = acre_tr_view(a, p->bn2_weight, p->bn2_bias, n2, ws + L.hpre, ws + L.st2, ws + L.red0);
  const int C = a.C;
  const long long Fw = acre_feat_width(C);
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_gather_kernel(cv); });
  cuda_emu::launch(dim3(1), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part0, Q, B, 1, (float)ACRE_PIX, p->bn0_eps, p->bn0_momentum, a.st0, p->bn0_mean,
                             p->bn0_var);
  });
  if (!a.par) {
    cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_THREADS), [&] { acre_tr_serial_kernel(a); });
  } else {
    cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_GATE_THREADS), [&] { acre_tr_gate_kernel(a); });
    run_gemm<EPI_STORE>(acre_plan_gate(a.gate, p->W_gate_e_weight, p->W_gate_e_bias, Q * C, a.y, 0));
  }
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { acre_tr_bn1_part_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(C, 256)), dim3(256), [&] {
    conve_tr_bn_stats_kernel(a.part1, Q, B, C, (float)ACRE_PIX, p->bn1_eps, p->bn1_momentum, a.st1, p->bn1_mean,
                             p->bn1_var);
  });
  cuda_emu::launch(dim3(proj_tiles(Q * Fw, 256)), dim3(256), [&] { acre_tr_feat_kernel(a); });
  float* partial = ws + L.partial;
  run_gemm<EPI_STORE>(conve_plan_fc(a.feat, p->fc_weight, Q, Fw, ACRE_K, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * ACRE_K, 256)), dim3(256), [&] {
    conve_tr_fc_combine_kernel(partial, conve_fc_slices(Fw), Q * ACRE_K, ACRE_K, p->fc_bias, n2, cv.hpre);
  });
  cuda_emu::launch(dim3(proj_tiles(ACRE_K, 256)), dim3(256), [&] {
    conve_tr_bn2_kernel(cv, p->bn2_eps, p->bn2_momentum, p->bn2_mean, p->bn2_var, x);
  });
}

void emu_acre_train_bwd(const kge_acre_train_t* p, const int64_t* e, const int64_t* r, int64_t Q, int64_t B,
                        const float* n0, const float* n1, const float* n2, const float* gx, const float* x,
                        float* const* grads, float* ws) {
  const AcreTrain a = args(p, e, r, Q, B, n0, n1, ws);
  const AcreTrainLayout L = acre_train_layout(Q, B, a.C, a.par);
  const ConveTrain cv = acre_tr_view(a, p->bn2_weight, p->bn2_bias, n2, ws + L.hpre, ws + L.st2, ws + L.red0);
  const int C = a.C;
  const long long Fw = acre_feat_width(C);
  float* dh = ws + L.dh;
  cuda_emu::launch(dim3(proj_tiles(ACRE_K, 256)), dim3(256),
                   [&] { conve_tr_bn2_bwd_kernel(cv, gx, x, dh, grads[16], grads[17], grads[15]); });
  run_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(dh, a.feat, Q, Fw, ACRE_K, grads[14]));
  run_gemm<EPI_STORE>(conve_plan_grad_feat(dh, p->fc_weight, Q, Fw, ACRE_K, a.feat));
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { acre_tr_bn1_bwd_part_kernel(a); });
  cuda_emu::launch(dim3(proj_tiles(C, 256)), dim3(256),
                   [&] { conve_tr_reduce_kernel(a.part1, Q, B, C, a.red1, grads[12], grads[13]); });
  cuda_emu::launch(dim3(proj_tiles(Q * Fw, 256)), dim3(256), [&] { acre_tr_bn1_bwd_kernel(a); });
  if (!a.par) {
    cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_THREADS), [&] { acre_tr_serial_bwd_kernel(a); });
  } else {
    const long long rows = Q * C;
    run_gemm<EPI_ATOMIC>(conve_plan_grad_fc_w(a.feat, a.gate, rows, ACRE_GATE, ACRE_PIX, grads[10]));
    cuda_emu::launch(dim3(proj_tiles(ACRE_PIX, 256)), dim3(256),
                     [&] { conve_tr_colsum_kernel(a.feat, rows, ACRE_PIX, grads[11]); });
    run_gemm<EPI_STORE>(conve_plan_grad_feat(a.feat, p->W_gate_e_weight, rows, ACRE_GATE, ACRE_PIX, a.gate));
    cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_GATE_THREADS), [&] { acre_tr_gate_bwd_kernel(a); });
  }
  for (int l = 0; l < 3; ++l) {
    const int nw = C * acre_tr_cin(l, C, a.par) * 9;
    cuda_emu::launch(dim3(proj_tiles(nw, 256)), dim3(256),
                     [&] { conve_tr_colsum_kernel(a.pw[l], Q, nw, grads[4 + 2 * l]); });
    if (a.has_bias)
      cuda_emu::launch(dim3(proj_tiles(C, 256)), dim3(256),
                       [&] { conve_tr_colsum_kernel(a.pb[l], Q, C, grads[5 + 2 * l]); });
  }
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { acre_tr_bn0_part_kernel(a); });
  cuda_emu::launch(dim3(1), dim3(256), [&] { conve_tr_reduce_kernel(a.part0, Q, B, 1, cv.red0, grads[2], grads[3]); });
  cuda_emu::launch(dim3((unsigned)Q), dim3(CONVE_TR_THREADS), [&] { conve_tr_bn0_bwd_kernel(cv, grads[0], grads[1]); });
}

}  // extern "C"

#ifdef ACRE_TRAIN_RACE_MAIN
// ThreadSanitizer build: the CTA-per-query kernels pass v, the conv maps, the weight banks (the serial backward's two
// map slots swapping roles across its three layers) and the CTA sums through shared memory and __syncthreads; both
// ways, two groups of two queries sharing an entity and a relation
static void run_way(int way, int C, bool bias) {
  const int N = 5, R = 3, B = 2, Q = 4, Fw = C * 400, cin = way == 0 ? C : 1;
  std::mt19937 gen(7 + way);
  std::normal_distribution<float> nd(0.f, 0.5f);
  auto rnd = [&](size_t n) { std::vector<float> v(n); for (auto& y : v) y = nd(gen); return v; };
  auto ent = rnd(N * 200), rel = rnd(2 * R * 200), fw = rnd((size_t)200 * Fw), fb = rnd(200);
  auto c1 = rnd(C * 9), c2 = rnd(C * cin * 9), c3 = rnd(C * cin * 9), cb1 = rnd(C), cb2 = rnd(C), cb3 = rnd(C);
  auto gw = rnd(400 * 1600), gb = rnd(400);
  auto gx = rnd(Q * 200), n0 = rnd(Q * 400), n1 = rnd(Q * C), n2 = rnd(Q * 200);
  std::vector<float> w0(1, 1.1f), b0(1, 0.1f), w1(C, 0.9f), b1(C, 0.05f), w2(200, 1.2f), b2(200, -0.1f);
  std::vector<float> rm0(1, 0.f), rv0(1, 1.f), rm1(C, 0.f), rv1(C, 1.f), rm2(200, 0.f), rv2(200, 1.f);
  kge_acre_train_t p{C, way, 1, 2, 3, 200, 2 * R, 1e-5f, 1e-5f, 1e-5f, 0.1f, 0.1f, 0.1f, ent.data(), rel.data(),
                     w0.data(), b0.data(), c1.data(), bias ? cb1.data() : nullptr, c2.data(),
                     bias ? cb2.data() : nullptr, c3.data(), bias ? cb3.data() : nullptr,
                     way ? gw.data() : nullptr, way ? gb.data() : nullptr, w1.data(), b1.data(), fw.data(), fb.data(),
                     w2.data(), b2.data(), rm0.data(), rv0.data(), rm1.data(), rv1.data(), rm2.data(), rv2.data()};
  std::vector<int64_t> e = {4, 1, 4, 0}, r = {2, 0, 2, 1};
  std::vector<float> ws(emu_acre_train_workspace_floats(&p, Q, B)), x(Q * 200);
  const size_t sizes[KGE_ACRE_TRAIN_GRADS] = {(size_t)N * 200, (size_t)2 * R * 200, 1, 1, (size_t)C * 9, (size_t)C,
                                              (size_t)C * cin * 9, (size_t)C, (size_t)C * cin * 9, (size_t)C,
                                              400 * 1600, 400, (size_t)C, (size_t)C, (size_t)200 * Fw, 200, 200, 200};
  std::vector<std::vector<float>> g(KGE_ACRE_TRAIN_GRADS);
  float* gp[KGE_ACRE_TRAIN_GRADS];
  for (int i = 0; i < KGE_ACRE_TRAIN_GRADS; ++i) {
    const bool absent = ((i == 5 || i == 7 || i == 9) && !bias) || ((i == 10 || i == 11) && !way);
    g[i].assign(absent ? 0 : sizes[i], 0.f);
    gp[i] = absent ? nullptr : g[i].data();
  }
  emu_acre_train_fwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), x.data(), ws.data());
  emu_acre_train_bwd(&p, e.data(), r.data(), Q, B, n0.data(), n1.data(), n2.data(), gx.data(), x.data(), gp,
                     ws.data());
  printf("%g %g\n", x[0], g[0][200]);
}

int main(int argc, char**) {
  if (argc > 1) return 64;   // "probe": only the sanitizer runtime starts
  run_way(0, 9, true);
  run_way(1, 3, false);
  return 0;
}
#endif
