// tests/emu/race_check_hyper.cpp — TEST INFRASTRUCTURE: data-race check of HypER's inference-trunk kernels
// (kge_hyper.cuh: filter GEMM, feature kernel, sliced Linear GEMM, combine) under the host emulation
// (tests/emu/cuda_runtime.h: one host thread per CUDA thread; __syncthreads is the only happens-before edge
// between them) in a binary built with -fsanitize=thread.  A missing barrier between a shared-memory write
// and another thread's read is reported by ThreadSanitizer and fails tests/test_emu_hyper.py; the same
// source built with -DCUDA_EMU_NO_BARRIERS must be reported (positive control).
//
//   race_check_hyper trunk
#include <cstdio>
#include <random>
#include <string>

#include "kge_hyper.cuh"

namespace cuda_emu {
thread_local dim3 t_threadIdx, t_blockIdx;
dim3 g_blockDim, g_gridDim;
BlockCtx* g_block = nullptr;
std::mutex g_atomic_mu;
}  // namespace cuda_emu

namespace kge {
void set_error(const char*, ...) {}
int cuda_fail(cudaError_t, const char*) { return KGE_ECUDA; }
void count_launch(int) {}
int sm_count() { return 132; }
}  // namespace kge

using namespace kge;

static std::vector<float> rnd(size_t n, unsigned seed, float scale = 0.5f, bool positive = false) {
  std::mt19937 g(seed);
  std::normal_distribution<float> d(0.f, scale);
  std::vector<float> v(n);
  for (auto& x : v) { x = d(g); if (positive) x = std::fabs(x) + 0.1f; }
  return v;
}

static void run_store_gemm(const ProjLaunch& L) {
  cuda_emu::launch(dim3(L.gx, L.gy, L.gz), dim3(PTHREADS), [&] { proj_gemm_kernel<EPI_STORE, 4, 4>(L.g); });
}

static int run_trunk() {
  const int de = 40, dr = 24; const long long Q = 5, N = 30, R = 4;
  const long long F = hyper_feat_width(de);
  const HyperLayout lay = hyper_layout(R, Q, de);
  auto ent = rnd(N * de, 1), rel = rnd(R * dr, 2), w1 = rnd(HYPER_FILT * dr, 3, 0.2f), b1 = rnd(HYPER_FILT, 4);
  auto fw = rnd(de * F, 5, 0.05f), fb = rnd(de, 6);
  auto b0w = rnd(1, 7, 1.f, true), b0b = rnd(1, 8), b0m = rnd(1, 9), b0v = rnd(1, 10, 1.f, true);
  auto b1w = rnd(32, 11, 1.f, true), b1b = rnd(32, 12), b1m = rnd(32, 13), b1v = rnd(32, 14, 1.f, true);
  auto b2w = rnd(de, 15, 1.f, true), b2b = rnd(de, 16), b2m = rnd(de, 17), b2v = rnd(de, 18, 1.f, true);
  std::vector<int64_t> e = {1, 5, 29, 0, 7}, r = {0, 3, 3, 2, 1};
  std::vector<float> ws(lay.total), x(Q * de);
  run_store_gemm(hyper_plan_filters(rel.data(), w1.data(), b1.data(), R, dr, ws.data() + lay.filt));
  HyperFeat f{};
  f.ent = ent.data(); f.filt = ws.data() + lay.filt; f.e = e.data(); f.r = r.data(); f.de = de;
  f.bn0_w = b0w.data(); f.bn0_b = b0b.data(); f.bn0_mean = b0m.data(); f.bn0_var = b0v.data(); f.bn0_eps = 1e-5f;
  f.bn1_w = b1w.data(); f.bn1_b = b1b.data(); f.bn1_mean = b1m.data(); f.bn1_var = b1v.data(); f.bn1_eps = 1e-5f;
  f.feat = ws.data() + lay.feat;
  cuda_emu::launch(dim3((unsigned)Q), dim3(HYPER_THREADS), [&] { hyper_feature_kernel(f); });
  float* partial = ws.data() + lay.partial;
  run_store_gemm(conve_plan_fc(f.feat, fw.data(), Q, F, de, partial));
  cuda_emu::launch(dim3(proj_tiles(Q * de, 256)), dim3(256), [&] {
    hyper_fc_combine_kernel(partial, conve_fc_slices(F), Q * de, de, fb.data(), b2w.data(), b2b.data(), b2m.data(),
                            b2v.data(), 1e-5f, x.data());
  });
  return 0;
}

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "trunk") return run_trunk();
  fprintf(stderr, "usage: race_check_hyper trunk\n");
  return 64;
}
