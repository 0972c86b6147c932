// tests/emu/race_check_interacte.cpp — TEST INFRASTRUCTURE: data-race check of InteractE's feature kernel
// (kge_interacte.cuh: filter bank, bn1 folds and padded images staged in shared memory, then the circular
// convolution) under the host emulation (tests/emu/cuda_runtime.h: one host thread per CUDA thread;
// __syncthreads is the only happens-before edge between them) in a binary built with -fsanitize=thread.
// A missing barrier between a shared-memory write and another thread's read is reported by ThreadSanitizer and
// fails tests/test_emu_interacte.py; the same source built with -DCUDA_EMU_NO_BARRIERS must be reported
// (positive control).
//
//   race_check_interacte features
#include <cstdio>
#include <random>
#include <string>

#include "kge_interacte.cuh"

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

static int run_features() {
  // P = 3 (odd and even images), F = 10 (a padded filter group), ks = 5 (pad 2), 8 x 6 images
  const int P = 3, F = 10, ks = 5, rh = 6, rw = 4, H = 2 * rw, W = rh, k = rh * rw;
  const long long Q = 3, N = 20, R = 4;
  std::mt19937 g(99);
  std::vector<int64_t> perm(P * 2 * k);
  for (int p = 0; p < P; ++p) {
    for (int i = 0; i < 2 * k; ++i) perm[p * 2 * k + i] = i;
    std::shuffle(perm.begin() + p * 2 * k, perm.begin() + (p + 1) * 2 * k, g);
  }
  auto ent = rnd(N * k, 1), rel = rnd(R * k, 2), filt = rnd(F * ks * ks, 3, 0.2f);
  auto b0w = rnd(P, 7, 1.f, true), b0b = rnd(P, 8), b0m = rnd(P, 9), b0v = rnd(P, 10, 1.f, true);
  auto b1w = rnd(P * F, 11, 1.f, true), b1b = rnd(P * F, 12), b1m = rnd(P * F, 13), b1v = rnd(P * F, 14, 1.f, true);
  std::vector<int64_t> e = {1, 19, 0}, r = {0, 3, 2};
  std::vector<float> feat(Q * interacte_feat_width(P, F, H, W));
  InteracteFeat f{};
  f.ent = ent.data(); f.rel = rel.data(); f.perm = perm.data(); f.e = e.data(); f.r = r.data();
  f.P = P; f.F = F; f.ks = ks; f.H = H; f.W = W;
  f.bn0_w = b0w.data(); f.bn0_b = b0b.data(); f.bn0_mean = b0m.data(); f.bn0_var = b0v.data(); f.bn0_eps = 1e-5f;
  f.conv_filt = filt.data();
  f.bn1_w = b1w.data(); f.bn1_b = b1b.data(); f.bn1_mean = b1m.data(); f.bn1_var = b1v.data(); f.bn1_eps = 1e-5f;
  f.feat = feat.data();
  cuda_emu::launch(dim3((unsigned)Q), dim3(INTERACTE_THREADS), [&] { interacte_feature_kernel(f); });
  return 0;
}

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "features") return run_features();
  fprintf(stderr, "usage: race_check_interacte features\n");
  return 64;
}
