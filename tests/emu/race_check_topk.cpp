// tests/emu/race_check_topk.cpp — TEST INFRASTRUCTURE: data-race check of the top-k row selection
// (kge_topk.cuh: the shared-memory row copy, the filter bitmap, the radix histograms and their block scans, the
// ordered tie compaction and the bitonic sort) under the host emulation (tests/emu/cuda_runtime.h: one host
// thread per CUDA thread; __syncthreads and the shuffles are the only happens-before edges between them) in a
// binary built with -fsanitize=thread.  A missing barrier between a shared-memory write and another thread's
// read is reported by ThreadSanitizer and fails tests/test_emu_topk.py; the same source built with
// -DCUDA_EMU_NO_BARRIERS must be reported (positive control).
//
//   race_check_topk select
#include <cstdio>
#include <string>

#include "cuda_runtime.h"

inline unsigned atomicOr(unsigned* p, unsigned v) { return __atomic_fetch_or(p, v, __ATOMIC_SEQ_CST); }

#include "kge_topk.cuh"

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
int num_tables(int) { return 0; }
}  // namespace kge

using namespace kge;

static int run_select() {
  // two rows of 700 candidates drawn from 9 values: the tie group at the threshold is larger than what is taken,
  // so the ordered compaction runs; row 1 has a filter with duplicates
  const int64_t n = 700, rows = 2;
  const int k = 40;
  std::vector<float> s(rows * n);
  for (int64_t i = 0; i < rows * n; ++i) s[i] = (float)((i * 7919) % 9) - 4.0f;
  std::vector<int64_t> ptr = {0, 0, 6}, idx = {3, 3, 650, 12, 699, 12};
  std::vector<int64_t> ids(rows * k);
  std::vector<float> out(rows * k);
  const TopkSelectPlan plan = topk_select_plan(n);
  const TopkSelectArgs A{s.data(), n, k, false, ptr.data(), idx.data(), ids.data(), out.data()};
  if (!plan.row_in_smem) return 2;
  cuda_emu::launch(dim3((unsigned)rows), dim3(kTopkThreads), [&] { topk_select_kernel<true>(A); });
  return 0;
}

int main(int argc, char** argv) {
  const std::string cmd = argc > 1 ? argv[1] : "";
  if (cmd == "select") return run_select();
  fprintf(stderr, "usage: race_check_topk select\n");
  return 64;
}
