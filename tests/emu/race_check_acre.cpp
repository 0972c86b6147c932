// tests/emu/race_check_acre.cpp — TEST INFRASTRUCTURE: data-race check of AcrE's serial feature kernel
// (kge_acre.cuh: image, bn1 folds and each layer's weight bank staged in shared memory, three convolutions
// chained through two shared-memory maps, five barriers) under the host emulation (tests/emu/cuda_runtime.h:
// one host thread per CUDA thread; __syncthreads is the only happens-before edge between them) in a binary
// built with -fsanitize=thread.  A missing barrier between a shared-memory write and another thread's read is
// reported by ThreadSanitizer and fails tests/test_emu_acre.py; the same source built with
// -DCUDA_EMU_NO_BARRIERS must be reported (positive control).
//
//   race_check_acre serial
#include <cstdio>
#include <random>
#include <string>

#include "kge_acre.cuh"

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

static int run_serial() {
  // C = 9: two channel groups, the second padded; rates 1 / 3 / 7 put taps in the padding at every layer
  const int C = 9;
  const long long Q = 2, N = 12, R2 = 6;
  auto ent = rnd(N * ACRE_K, 1), rel = rnd(R2 * ACRE_K, 2);
  auto w1 = rnd(C * 9, 3, 0.3f), w2 = rnd(C * C * 9, 4, 0.1f), w3 = rnd(C * C * 9, 5, 0.1f);
  auto b1 = rnd(C, 6), b2 = rnd(C, 7), b3 = rnd(C, 8);
  auto b0w = rnd(1, 9, 1.f, true), b0b = rnd(1, 10), b0m = rnd(1, 11), b0v = rnd(1, 12, 1.f, true);
  auto b1w = rnd(C, 13, 1.f, true), b1b = rnd(C, 14), b1m = rnd(C, 15), b1v = rnd(C, 16, 1.f, true);
  std::vector<int64_t> e = {3, 0}, r = {0, 5};
  std::vector<float> feat(Q * acre_feat_width(C));
  AcreFeat f{};
  f.ent = ent.data(); f.rel = rel.data(); f.e = e.data(); f.r = r.data(); f.C = C;
  f.dil[0] = 1; f.dil[1] = 3; f.dil[2] = 7;
  f.bn0_w = b0w.data(); f.bn0_b = b0b.data(); f.bn0_mean = b0m.data(); f.bn0_var = b0v.data(); f.bn0_eps = 1e-5f;
  f.conv_w[0] = w1.data(); f.conv_w[1] = w2.data(); f.conv_w[2] = w3.data();
  f.conv_b[0] = b1.data(); f.conv_b[1] = b2.data(); f.conv_b[2] = b3.data();
  f.bn1_w = b1w.data(); f.bn1_b = b1b.data(); f.bn1_mean = b1m.data(); f.bn1_var = b1v.data(); f.bn1_eps = 1e-5f;
  f.out = feat.data();
  cuda_emu::launch(dim3((unsigned)Q), dim3(ACRE_THREADS), [&] { acre_serial_feature_kernel(f); });
  return 0;
}

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "serial") return run_serial();
  fprintf(stderr, "usage: race_check_acre serial\n");
  return 64;
}
