// kge_rank_tc.cuh — device helpers shared by the tensor-core sweep (kge_rank_tc.cu) and the kernels
// that prepare its operands inside the fp32 path's preparation kernels (kge_rank_tiled.cu).
#pragma once
#include <cuda_bf16.h>

#include "kge_common.cuh"

namespace kge {

// Per-direction outputs of the query preparation for the tensor-core level (A0 == nullptr: disabled).
struct TcQueryArgs {
  __nv_bfloat16* A0;          // [Q][Kp] bf16 high parts of the query vectors (+ the -1 norm columns)
  __nv_bfloat16* A1;          // [Q][Kp] bf16 low parts
  float* tau;                 // [Q][4] band of the accumulator test against candidate c with norm bound n_c:
                              //   centre, a, b, e :  half(q,c) = a + b n_c + e n_c^2 ;
                              //   certainly better: D - centre > half;  certainly not: D - centre < -half
  int32_t* tc_counts;         // [Q] zeroed here
  unsigned* ctrl;             // [4] zeroed here: pair-list length, overflow, done counter (+ 1 unused)
  int Kp, kind;               // padded contraction length; 0 dot, 1 squared distance (sum domain), 2 squared distance - margin
  float sign, margin;
};

KGE_DEV double tc_group_sum_d(double v) {
  const unsigned m = group_mask();
  v += __shfl_xor_sync(m, v, 4);
  v += __shfl_xor_sync(m, v, 2);
  v += __shfl_xor_sync(m, v, 1);
  return v;
}

// x -> (bf16_rn(x), bf16_rn(x - bf16_rn(x))) for the 4 elements of a chunk; |x - x0 - x1| <= 2^-18 |x|
KGE_DEV void tc_split_store(__nv_bfloat16* o0, __nv_bfloat16* o1, float4 x, float sign) {
  __nv_bfloat16 h[4], l[4];
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float xv = sign * f4_get(x, e);
    h[e] = __float2bfloat16_rn(xv);
    l[e] = __float2bfloat16_rn(__fsub_rn(xv, __bfloat162float(h[e])));   // xv - h is exact in fp32
  }
  *reinterpret_cast<uint2*>(o0) = *reinterpret_cast<const uint2*>(h);
  *reinterpret_cast<uint2*>(o1) = *reinterpret_cast<const uint2*>(l);
}

// columns [K, Kp) of an operand row: zero, except (first == true) the three norm columns n0 n1 n2
KGE_DEV void tc_store_tail(__nv_bfloat16* o0, __nv_bfloat16* o1, int K, int Kp, int lane, bool first,
                           __nv_bfloat16 n0, __nv_bfloat16 n1, __nv_bfloat16 n2) {
  for (int c = K / 4 + lane; c < Kp / 4; c += 8) {   // K and Kp are multiples of 4
    __nv_bfloat16 h[4], l[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { h[j] = __float2bfloat16_rn(0.f); l[j] = h[j]; }
    if (first && c == K / 4) { h[0] = n0; h[1] = n1; h[2] = n2; }
    *reinterpret_cast<uint2*>(o0 + 4 * c) = *reinterpret_cast<const uint2*>(h);
    *reinterpret_cast<uint2*>(o1 + 4 * c) = *reinterpret_cast<const uint2*>(l);
  }
}

// Called by the 8 lanes of a query's group once its fp32 query vectors src[0 .. K) (K = KQ * dp, zero
// padded, visible to the whole group) and its threshold th (the target's own canonical score) exist:
// writes the bf16 split of the vectors (sign -1 for the head sweep of the translational models, whose
// canonical distance is |c + q|), the -1 norm columns, and the coefficients of the accumulator band.
//
// Error budget PER PAIR (q, c) — in double, rounded outwards to float at the end.  n = |c| (an upper bound,
// written per candidate row by tc_prep_cand_kernel), A = |q| n >= sum_k |q_k c_k|,
// M = A (+ n^2 / 2 when the norm columns ride along) bounds every partial sum of the accumulation.
//   split      : |x - x0 - x1| <= 2^-18 |x| per operand; the three dropped product terms
//                (a1 b1, da b, a db) are <= 3 * 2^-18 * (1 + 2^-8) A                      -> 2^-16 A  (x 1.33 slack)
//   accumulate : products of bf16 pairs are exact in fp32; each of the nmma = 3 ceil(Kp/16) tensor-core
//                instructions may lose <= 4 ulp of the running magnitude                   -> nmma 2^-21 M
//   norm cols  : 3-way bf16 split of fl(|c|^2 / 2)                                         -> 2^-22 n^2
//   canonical  : the fp32 chain (RSUM: 8 partials of K/8 fma + 3 butterfly adds; squared distances add one
//                rounding of (q - c) per element) against the exact value of the same fp32 operands:
//                gamma = (K/8 + 8) 2^-24 (+ 2^-22), times A (dot) or (|q| + n)^2 (distance).
// Every term is a polynomial of degree <= 2 in n with per-query coefficients, so the epilogue evaluates
// half(q,c) = a + b n + e n^2 with two fma (r2 first used max_c|c| for n: exact too, but one heavy row —
// trained tables have them — widened every pair's band; now the band of a pair scales with ITS candidate).
// tests/test_gpu_baseline_shapes.py measures the real error against this bound at every BASELINE shape.
KGE_DEV void tc_query_finish(const TcQueryArgs& T, const float* src, float th, int64_t q, int lane, int K) {
  __nv_bfloat16* o0 = T.A0 + (size_t)q * T.Kp;
  __nv_bfloat16* o1 = T.A1 + (size_t)q * T.Kp;
  double ss = 0.0;
  for (int c = lane; c < K / 4; c += 8) {
    const float4 x = *(reinterpret_cast<const float4*>(src) + c);
#pragma unroll
    for (int j = 0; j < 4; ++j) ss += (double)f4_get(x, j) * (double)f4_get(x, j);
    tc_split_store(o0 + 4 * c, o1 + 4 * c, x, T.sign);
  }
  ss = tc_group_sum_d(ss);
  const __nv_bfloat16 m1 = __float2bfloat16_rn(-1.0f);
  tc_store_tail(o0, o1, K, T.Kp, lane, T.kind != 0, m1, m1, m1);
  if (lane != 0) return;
  T.tc_counts[q] = 0;
  const double nq = sqrt(ss) * (1.0 + 1e-7);
  const int nmma = 3 * ((T.Kp + 15) / 16);
  const double acc = (double)nmma * ldexp(1.0, -21);
  const double gamma = ((double)K / 8.0 + 8.0) * ldexp(1.0, -24);
  double centre, a, b, e;
  if (T.kind == 0) {
    centre = -(double)th;                        // canonical: -sum < th  <=>  sum > -th (negation is exact)
    a = 0.0;
    b = nq * (ldexp(1.0, -16) + acc + gamma);
    e = 0.0;
  } else {
    // e_tc = 2^-16 nq n + acc (nq n + n^2/2) + 2^-22 n^2 ;  smax = (nq + n)^2 = nq^2 + 2 nq n + n^2
    const double g2 = gamma + ldexp(1.0, -22);
    double ks = 0.5 * g2;                        // coefficient of smax in the half band
    double a0 = ldexp(1.0, -50) * ss;
    if (T.kind == 1) {                           // canonical: sum < T(th)
      const double Tt = (double)sqrt_domain_threshold(th);
      centre = 0.5 * (ss - Tt);
    } else {                                     // canonical: fsub(sum, margin) < th
      centre = 0.5 * (ss - (double)th - (double)T.margin);
      ks += 0.5 * 1.01 * ldexp(1.0, -24);        // the rounding of fsub(sum, margin)
      a0 += 0.5 * ldexp(1.0, -24) * fabs((double)T.margin);
    }
    a = a0 + ks * nq * nq;
    b = nq * (ldexp(1.0, -16) + acc) + 2.0 * ks * nq;
    e = 0.5 * acc + ldexp(1.0, -22) + ks;
  }
  // The epilogue evaluates u = fsub(D, centre_f) and half = fma(fma(e, n, b), n, a) in fp32: cover the
  // rounding of centre to float (2^-24 |centre|, absolute), of u (2^-24 relative — harmless against the
  // 2^-18 inflation) and of the two fma (2^-23 relative).
  const double infl = 1.0 + ldexp(1.0, -18);
  a = a * infl + ldexp(1.0, -23) * fabs(centre) + 1e-30;
  // NaN thresholds propagate: every comparison with them is false, as `s < NaN` is in the exact path
  float4 o;
  o.x = (float)centre;
  o.y = __double2float_ru(a);
  o.z = __double2float_ru(b * infl);
  o.w = __double2float_ru(e * infl);
  *reinterpret_cast<float4*>(T.tau + 4 * q) = o;
}

}  // namespace kge
