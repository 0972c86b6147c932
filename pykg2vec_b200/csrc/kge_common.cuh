// kge_common.cuh — shared device/host helpers of libkge_b200.so (sm_90a only).
//
// Canonical arithmetic (DESIGN.md §3): every score is evaluated with explicitly
// rounded fp32 intrinsics (__fmaf_rn/__fadd_rn/__fmul_rn: never contracted or
// re-associated by nvcc), reductions over the embedding axis use the RSUM order:
// 8 partial sums, element j -> partial (j>>2)&7 in increasing j, combined by the
// xor butterfly 4,2,1.  An 8-lane group evaluates one (h,r,t) triple: lane l owns
// the 4-element chunks c = l, l+8, l+16, ... so each lane's register accumulator
// IS partial l, and the butterfly is three __shfl_xor_sync steps.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "../../include/kge_b200.h"

namespace kge {

// ---- host side: error reporting / launch accounting --------------------------
void set_error(const char* fmt, ...);
int cuda_fail(cudaError_t e, const char* what);
void count_launch(int n = 1);
int sm_count();

#define KGE_CUDA_OK(expr)                                   \
  do {                                                      \
    cudaError_t _e = (expr);                                \
    if (_e != cudaSuccess) return ::kge::cuda_fail(_e, #expr); \
  } while (0)

#define KGE_CHECK_LAUNCH(name)                                  \
  do {                                                          \
    ::kge::count_launch();                                      \
    cudaError_t _e = cudaGetLastError();                        \
    if (_e != cudaSuccess) return ::kge::cuda_fail(_e, name);   \
  } while (0)

// Largest vector width (in floats) usable for row loads of width `d` from the tables
// tabs[0 .. ntab) when their base pointers are all aligned accordingly.
inline int pick_vec(const float* const* tabs, int ntab, int d, int d2 = 0) {
  int vec = 4;
  if (d % 4 != 0 || (d2 && d2 % 4 != 0)) vec = (d % 2 == 0 && (!d2 || d2 % 2 == 0)) ? 2 : 1;
  for (int k = 0; k < ntab; ++k) {
    const uintptr_t a = (uintptr_t)tabs[k];
    if (vec == 4 && (a & 15)) vec = 2;
    if (vec == 2 && (a & 7)) vec = 1;
  }
  return vec;
}
inline int pick_vec(const kge_model_t* m, int ntab, int d, int d2 = 0) { return pick_vec(m->tables, ntab, d, d2); }

// ---- device side ---------------------------------------------------------------
#define KGE_DEV __device__ __forceinline__

KGE_DEV float fmul(float a, float b) { return __fmul_rn(a, b); }
KGE_DEV float fadd(float a, float b) { return __fadd_rn(a, b); }
KGE_DEV float fsub(float a, float b) { return __fsub_rn(a, b); }
KGE_DEV float ffma(float a, float b, float c) { return __fmaf_rn(a, b, c); }

// RSUM butterfly across the 8 lanes of a group.  The shuffle mask names only the
// group's own lanes, so different groups of a warp may diverge freely.
KGE_DEV unsigned group_mask() { return 0xFFu << (threadIdx.x & 24); }
KGE_DEV float group_sum(float v) {
  const unsigned m = group_mask();
  v = fadd(v, __shfl_xor_sync(m, v, 4));
  v = fadd(v, __shfl_xor_sync(m, v, 2));
  v = fadd(v, __shfl_xor_sync(m, v, 1));
  return v;
}

// 1 / max(sqrt(sumsq), 1e-12)  — F.normalize(eps=1e-12) as a reciprocal multiply
KGE_DEV float inv_norm_from_sumsq(float sumsq) {
  return __frcp_rn(fmaxf(__fsqrt_rn(sumsq), 1e-12f));
}

// Plain L2 distances are compared in the SUM domain (DESIGN.md §3 rule 7): sqrt_rn is monotone, so
//   sqrt_rn(sum) < th   <=>   sum < T(th),   T(th) = min{x >= 0 : sqrt_rn(x) >= th},
// and T is found exactly by walking a few ulps around th*th.  Saves the IEEE square root per
// (query, candidate) pair without changing a single comparison result.
KGE_DEV float sqrt_domain_threshold(float th) {
  if (!(th > 0.f)) return 0.f;                       // sqrt(.) >= 0 is never below th (also th = NaN)
  float x = fmul(th, th);                            // may round to +inf or to 0
  while (__fsqrt_rn(x) >= th) x = __uint_as_float(__float_as_uint(x) - 1u);  // never reaches below +0: sqrt(0) < th
  while (__fsqrt_rn(x) < th) x = __uint_as_float(__float_as_uint(x) + 1u);   // stops at +inf at the latest
  return x;
}

// Canonical sin/cos: Cody-Waite by pi/2 (3 parts) + Cephes minimax polynomials,
// written with explicit fma so that it is bit-identical to oracle/kge_oracle.c.
KGE_DEV void sincos_canon(float x, float& sn, float& cs) {
  const float k = rintf(fmul(x, 0.636619772367581343f));
  float r = ffma(-k, 1.57079601287841796875f, x);
  r = ffma(-k, 3.13916473303834209219e-7f, r);
  r = ffma(-k, 5.39030252995776476554e-15f, r);
  const float s = fmul(r, r);
  float ps = ffma(s, -1.9515295891e-4f, 8.3321608736e-3f);
  ps = ffma(s, ps, -1.6666654611e-1f);
  const float sr = ffma(fmul(r, s), ps, r);
  float pc = ffma(s, 2.443315711809948e-5f, -1.388731625493765e-3f);
  pc = ffma(s, pc, 4.166664568298827e-2f);
  const float cr = ffma(fmul(s, s), pc, ffma(s, -0.5f, 1.0f));
  const int q = ((int)k) & 3;
  const float so = (q & 1) ? cr : sr;
  const float co = (q & 1) ? sr : cr;
  sn = (q & 2) ? -so : so;
  cs = ((q + 1) & 2) ? -co : co;
}

// Canonical exp / sigmoid (Cephes expf in explicit fma; bit-identical to oracle/kge_oracle.c)
KGE_DEV float exp_canon(float x) {
  x = fminf(fmaxf(x, -87.0f), 87.0f);
  const float k = rintf(fmul(x, 1.44269504088896341f));
  float r = ffma(-k, 0.693359375f, x);
  r = ffma(-k, -2.12194440e-4f, r);
  float p = ffma(r, 1.9875691500e-4f, 1.3981999507e-3f);
  p = ffma(p, r, 8.3334519073e-3f);
  p = ffma(p, r, 4.1665795894e-2f);
  p = ffma(p, r, 1.6666665459e-1f);
  p = ffma(p, r, 5.0000001201e-1f);
  const float y = fadd(ffma(p, fmul(r, r), r), 1.0f);
  return fmul(y, __uint_as_float((unsigned)((int)k + 127) << 23));
}
KGE_DEV float sigmoid_canon(float x) { return __frcp_rn(fadd(1.0f, exp_canon(-x))); }

// Canonical tanh (Cephes tanhf; bit-identical to oracle/kge_oracle.c)
KGE_DEV float tanh_canon(float x) {
  const float ax = fabsf(x);
  if (ax < 0.625f) {
    const float z = fmul(x, x);
    float p = ffma(-5.70498872745e-3f, z, 2.06390887954e-2f);
    p = ffma(p, z, -5.37397155531e-2f);
    p = ffma(p, z, 1.33314422036e-1f);
    p = ffma(p, z, -3.33332819422e-1f);
    return ffma(fmul(p, z), x, x);
  }
  const float e = exp_canon(fmul(2.0f, ax));
  const float t = fsub(1.0f, fmul(2.0f, __frcp_rn(fadd(e, 1.0f))));
  return x < 0.0f ? -t : t;
}

// Canonical natural logarithm (Cephes logf in explicit fma; bit-identical to oracle/kge_oracle.c)
KGE_DEV float log_canon(float x) {
  if (!(x > 0.0f)) return x == 0.0f ? -INFINITY : NAN;
  if (isinf(x)) return x;
  int e = 0;
  if (x < 1.17549435e-38f) { x = fmul(x, 8388608.0f); e = -23; }
  unsigned u = __float_as_uint(x);
  e += (int)((u >> 23) & 0xff) - 126;
  float m = __uint_as_float((u & 0x007fffffu) | 0x3f000000u);
  if (m < 0.707106781186547524f) { e -= 1; m = fsub(fadd(m, m), 1.0f); } else { m = fsub(m, 1.0f); }
  const float z = fmul(m, m);
  float y = ffma(7.0376836292e-2f, m, -1.1514610310e-1f);
  y = ffma(y, m, 1.1676998740e-1f);
  y = ffma(y, m, -1.2420140846e-1f);
  y = ffma(y, m, 1.4249322787e-1f);
  y = ffma(y, m, -1.6668057665e-1f);
  y = ffma(y, m, 2.0000714765e-1f);
  y = ffma(y, m, -2.4999993993e-1f);
  y = ffma(y, m, 3.3333331174e-1f);
  y = fmul(fmul(y, m), z);
  const float fe = (float)e;
  y = ffma(-2.12194440e-4f, fe, y);
  y = ffma(-0.5f, z, y);
  float r = fadd(m, y);
  r = ffma(0.693359375f, fe, r);
  return r;
}

// One 4-element chunk c of a row of width d (elements 4c..4c+3; elements >= d read as 0,
// which is an exact identity for every accumulation used here).
template <int VEC>
KGE_DEV float4 ld_chunk(const float* __restrict__ row, int c, int d) {
  float4 v;
  if (VEC == 4) {
    v = __ldg(reinterpret_cast<const float4*>(row) + c);
  } else if (VEC == 2) {
    const int j = 4 * c;
    const float2 a = __ldg(reinterpret_cast<const float2*>(row + j));
    float2 b = make_float2(0.f, 0.f);
    if (j + 2 < d) b = __ldg(reinterpret_cast<const float2*>(row + j + 2));
    v = make_float4(a.x, a.y, b.x, b.y);
  } else {
    const int j = 4 * c;
    v.x = __ldg(row + j);
    v.y = (j + 1 < d) ? __ldg(row + j + 1) : 0.f;
    v.z = (j + 2 < d) ? __ldg(row + j + 2) : 0.f;
    v.w = (j + 3 < d) ? __ldg(row + j + 3) : 0.f;
  }
  return v;
}

// atomic accumulate of one chunk of a gradient row
template <int VEC>
KGE_DEV void red_chunk(float* __restrict__ row, int c, int d, float4 g) {
  const int j = 4 * c;
  if (VEC == 4) {
    atomicAdd(reinterpret_cast<float4*>(row) + c, g);
  } else {
    atomicAdd(row + j, g.x);
    if (j + 1 < d) atomicAdd(row + j + 1, g.y);
    if (j + 2 < d) atomicAdd(row + j + 2, g.z);
    if (j + 3 < d) atomicAdd(row + j + 3, g.w);
  }
}

KGE_DEV float& f4_at(float4& v, int e) { return reinterpret_cast<float*>(&v)[e]; }
KGE_DEV float f4_get(const float4& v, int e) { return reinterpret_cast<const float*>(&v)[e]; }

// Per-model constants handed to the kernels by value.
struct ModelParams {
  const float* tab[KGE_MAX_TABLES];   // candidate-side / default tables
  const float* qtab[KGE_MAX_TABLES];  // query-side tables (== tab unless row-sharded)
  int d;          // entity width
  int dr;         // relation width
  int l1;         // TransE family
  float margin;   // RotatE
  float phase;    // RotatE phase scale
};

inline ModelParams make_params(const kge_model_t* m, const kge_model_t* mq) {
  ModelParams p;
  for (int k = 0; k < KGE_MAX_TABLES; ++k) {
    p.tab[k] = m->tables[k];
    p.qtab[k] = mq ? mq->tables[k] : m->tables[k];
  }
  p.d = m->dim; p.dr = m->rel_dim; p.l1 = m->l1_flag; p.margin = m->margin; p.phase = m->phase_scale;
  return p;
}

int num_tables(int model);

}  // namespace kge
