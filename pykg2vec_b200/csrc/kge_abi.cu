// kge_abi.cu — library info, error reporting, launch accounting (host only).
#include <atomic>
#include <cstdarg>
#include <cstdio>

#include "kge_common.cuh"

namespace kge {

static thread_local char g_err[512] = "";
static std::atomic<long long> g_launches{0};

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

int cuda_fail(cudaError_t e, const char* what) {
  set_error("CUDA error %d (%s) at %s", (int)e, cudaGetErrorString(e), what);
  return KGE_ECUDA;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

int sm_count() {
  // queried lazily (never at load time: the library must be fork-safe)
  static thread_local int cached = 0;
  if (cached) return cached;
  int dev = 0, n = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return 132;
  if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) return 132;
  cached = n;
  return n;
}

int num_tables(int model) {
  switch (model) {
    case KGE_TRANSE: case KGE_DISTMULT: case KGE_HOLE: case KGE_RESCAL: return 2;
    case KGE_TRANSH: case KGE_TRANSR: case KGE_ROTATE: case KGE_CP: case KGE_TRANSM: return 3;
    case KGE_TRANSD: case KGE_COMPLEX: case KGE_SIMPLE: case KGE_SIMPLE_IGNR: case KGE_KG2E: return 4;
    case KGE_ANALOGY: return 6;
    case KGE_QUATE: case KGE_SME: case KGE_SME_BL: return 8;
    case KGE_SLM: case KGE_CONVKB: return 4;
    case KGE_NTN: return 6;
    case KGE_OCTONIONE: return 16;
    default: return 0;
  }
}

}  // namespace kge

extern "C" {

int kge_abi_version(void) { return KGE_ABI_VERSION; }
const char* kge_version(void) { return "kge_b200 0.1 (sm_90a)"; }
const char* kge_last_error(void) { return kge::g_err; }
int64_t kge_launch_count(void) { return (int64_t)kge::g_launches.load(std::memory_order_relaxed); }

}  // extern "C"
