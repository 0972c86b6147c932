// tests/emu/cuda_runtime.h — TEST INFRASTRUCTURE: a host stand-in for <cuda_runtime.h>.
//
// There is no GPU in the build container.  To exercise the indexing / synchronisation logic of a
// CUDA kernel before it ever reaches a GPU, tests/emu/*.cpp compile the product's kernel headers
// (pykg2vec_b200/csrc/*.cuh) with g++ against THIS header (found first through -I tests/emu) and
// run every CUDA thread of a block as a host thread: __syncthreads() is a barrier over the block,
// __shfl_xor_sync an exchange among the lanes named by its mask, atomics are host atomics, and
// the rounding intrinsics map to the IEEE operations they denote (build with -ffp-contract=off).
// It models correctness only (no memory model subtleties, no timing); blocks run one at a time,
// so __shared__ variables are function-local statics.  A kernel thread that returns before a later
// __syncthreads() would hang the barrier (on the GPU exited threads leave the barrier count); none of
// the emulated kernels does that.
#pragma once
#include <math.h>
#include <pthread.h>
#include <stdint.h>
#include <string.h>

#include <algorithm>
#include <condition_variable>
#include <functional>
#include <map>
#include <mutex>
#include <thread>
#include <vector>

#define __global__ static
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __shared__ static
#define __launch_bounds__(...)
#define __align__(n) __attribute__((aligned(n)))

struct dim3 {
  unsigned x, y, z;
  dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
struct __attribute__((aligned(16))) float4 { float x, y, z, w; };
struct __attribute__((aligned(8))) float2 { float x, y; };
inline float4 make_float4(float x, float y, float z, float w) { return float4{x, y, z, w}; }
inline float2 make_float2(float x, float y) { return float2{x, y}; }

typedef int cudaError_t;
typedef void* cudaStream_t;
enum { cudaSuccess = 0 };
inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }

namespace cuda_emu {
struct WarpExchange {
  std::mutex mu;
  std::condition_variable cv;
  struct State { int arrived = 0, departed = 0, phase = 0; uint32_t vals[32]; };
  std::map<unsigned, State> st;
};
struct BlockCtx {
  pthread_barrier_t barrier;
  std::vector<WarpExchange> warps;
};
extern thread_local dim3 t_threadIdx, t_blockIdx;
extern dim3 g_blockDim, g_gridDim;
extern BlockCtx* g_block;
extern std::mutex g_atomic_mu;

inline int linear_tid() { return (int)(t_threadIdx.x + g_blockDim.x * (t_threadIdx.y + g_blockDim.y * t_threadIdx.z)); }

inline uint32_t shfl(unsigned mask, uint32_t val, int src_lane) {
  const int tid = linear_tid(), lane = tid & 31;
  WarpExchange& w = g_block->warps[tid >> 5];
  const int n = __builtin_popcount(mask);
  std::unique_lock<std::mutex> lk(w.mu);
  WarpExchange::State& s = w.st[mask];
  w.cv.wait(lk, [&] { return s.phase == 0; });
  s.vals[lane] = val;
  if (++s.arrived == n) { s.phase = 1; w.cv.notify_all(); }
  else w.cv.wait(lk, [&] { return s.phase == 1; });
  const uint32_t out = s.vals[src_lane & 31];
  if (++s.departed == n) { s.arrived = s.departed = 0; s.phase = 0; w.cv.notify_all(); }
  return out;
}

// run `body` once per CUDA thread of every block of the grid.  Blocks run one after the other (their
// __shared__ variables are function-local statics); the host threads are created once per launch and
// walk the blocks together, separated by the block barrier.
inline void launch(dim3 grid, dim3 block, const std::function<void()>& body) {
  g_gridDim = grid; g_blockDim = block;
  const int nthreads = (int)(block.x * block.y * block.z);
  BlockCtx ctx;
  pthread_barrier_init(&ctx.barrier, nullptr, nthreads);
  ctx.warps = std::vector<WarpExchange>((nthreads + 31) / 32);
  g_block = &ctx;
  std::vector<std::thread> th;
  th.reserve(nthreads);
  for (int t = 0; t < nthreads; ++t)
    th.emplace_back([&, t] {
      t_threadIdx = dim3(t % block.x, (t / block.x) % block.y, t / (block.x * block.y));
      for (unsigned bz = 0; bz < grid.z; ++bz)
        for (unsigned by = 0; by < grid.y; ++by)
          for (unsigned bx = 0; bx < grid.x; ++bx) {
            t_blockIdx = dim3(bx, by, bz);
            body();
            pthread_barrier_wait(&ctx.barrier);   // end of this block for every thread
          }
    });
  for (auto& x : th) x.join();
  pthread_barrier_destroy(&ctx.barrier);
  g_block = nullptr;
}
}  // namespace cuda_emu

#define threadIdx (::cuda_emu::t_threadIdx)
#define blockIdx (::cuda_emu::t_blockIdx)
#define blockDim (::cuda_emu::g_blockDim)
#define gridDim (::cuda_emu::g_gridDim)

// NOTE: a thread that returns early from a kernel that later calls __syncthreads() would hang a
// pthread barrier (on the GPU exited threads are dropped from the barrier count); none of the
// emulated kernels does that.
// CUDA_EMU_NO_BARRIERS: positive control of the race check (tests/test_emu_races.py) — with the block
// barrier compiled out ThreadSanitizer must report the shared-memory races it is there to find.
#ifdef CUDA_EMU_NO_BARRIERS
inline void __syncthreads() {}
#else
inline void __syncthreads() { pthread_barrier_wait(&::cuda_emu::g_block->barrier); }
#endif

template <class T> inline T __ldg(const T* p) { return *p; }
inline float __fmaf_rn(float a, float b, float c) { return fmaf(a, b, c); }
inline float __fadd_rn(float a, float b) { return a + b; }
inline float __fsub_rn(float a, float b) { return a - b; }
inline float __fmul_rn(float a, float b) { return a * b; }
inline float __fsqrt_rn(float a) { return sqrtf(a); }
inline float __frcp_rn(float a) { return 1.0f / a; }
inline float __fdiv_rn(float a, float b) { return a / b; }
inline float __uint_as_float(unsigned u) { float f; memcpy(&f, &u, 4); return f; }
inline unsigned __float_as_uint(float f) { unsigned u; memcpy(&u, &f, 4); return u; }
using std::max;
using std::min;

inline int __shfl_xor_sync(unsigned mask, int v, int lane_mask) {
  const int lane = ::cuda_emu::linear_tid() & 31;
  return (int)::cuda_emu::shfl(mask, (uint32_t)v, lane ^ lane_mask);
}
inline float __shfl_xor_sync(unsigned mask, float v, int lane_mask) {
  const int lane = ::cuda_emu::linear_tid() & 31;
  return __uint_as_float(::cuda_emu::shfl(mask, __float_as_uint(v), lane ^ lane_mask));
}

// warp barrier among the lanes named by the mask
inline void __syncwarp(unsigned mask = 0xffffffffu) { (void)::cuda_emu::shfl(mask, 0u, ::cuda_emu::linear_tid() & 31); }

inline int atomicAdd(int* p, int v) { return __atomic_fetch_add(p, v, __ATOMIC_SEQ_CST); }
inline int atomicSub(int* p, int v) { return __atomic_fetch_sub(p, v, __ATOMIC_SEQ_CST); }
inline float atomicAdd(float* p, float v) {
  std::lock_guard<std::mutex> lk(::cuda_emu::g_atomic_mu);
  const float old = *p;
  *p = old + v;
  return old;
}
inline float4 atomicAdd(float4* p, float4 v) {
  std::lock_guard<std::mutex> lk(::cuda_emu::g_atomic_mu);
  const float4 old = *p;
  p->x += v.x; p->y += v.y; p->z += v.z; p->w += v.w;
  return old;
}
