// tests/emu/race_check_proje.cpp — TEST INFRASTRUCTURE: data-race check of ProjE_pointwise's training-step kernel
// (kge_proje.cuh: the label-row scan, the compacted entry list and its flushes, d loss / d x in shared memory)
// under the host emulation (tests/emu/cuda_runtime.h: one host thread per CUDA thread; __syncthreads is the only
// happens-before edge between them) in a binary built with -fsanitize=thread.  A missing barrier between a
// shared-memory write and another thread's read is reported by ThreadSanitizer and fails tests/test_emu_proje.py;
// the same source built with -DCUDA_EMU_NO_BARRIERS must be reported (positive control).
//
//   race_check_proje step
#include <cstdio>
#include <random>
#include <string>

#include "kge_proje.cuh"

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

static std::vector<float> rnd(size_t n, unsigned seed, float scale = 0.3f) {
  std::mt19937 g(seed);
  std::normal_distribution<float> d(0.f, scale);
  std::vector<float> v(n);
  for (auto& x : v) x = d(g);
  return v;
}

static int run_step() {
  // N > PROJE_CAP with a dense label row: the entry list is flushed in the middle of the row
  const int k = 12, B = 2;
  const long long N = 2600, R = 3;
  auto ent = rnd(N * k, 1), rel = rnd(R * k, 2), vec = rnd(6 * k, 3);
  std::vector<float> lab(B * N, 0.f), gent(N * k, 0.f), grel(R * k, 0.f), gv(6 * k, 0.f), loss(1, 0.f);
  for (long long i = 0; i < B * N; ++i) lab[i] = (i % 3 == 0) ? 1.f : ((i % 3 == 1) ? -1.f : 0.f);
  std::vector<int64_t> h = {5, 2599}, r = {0, 2}, t = {17, 0};
  ProjeStep s{};
  s.ent = ent.data(); s.rel = rel.data(); s.r = r.data(); s.N = N; s.k = k; s.B = B;
  s.gent = gent.data(); s.grel = grel.data();
  const float* v = vec.data();
  float* g = gv.data();
  s.dir[0] = ProjeDir{h.data(), lab.data(), nullptr, v + k, v + 2 * k, v, g + k, g + 2 * k, g};
  s.dir[1] = ProjeDir{t.data(), lab.data(), nullptr, v + 4 * k, v + 5 * k, v + 3 * k, g + 4 * k, g + 5 * k, g + 3 * k};
  s.dirs[0] = 0; s.dirs[1] = 1;
  s.loss = loss.data();
  cuda_emu::launch(dim3(B, 2), dim3(PROJE_THREADS), [&] { proje_step_kernel(s); });
  return 0;
}

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "step") return run_step();
  fprintf(stderr, "usage: race_check_proje step\n");
  return 64;
}
