// kge_models.cuh — per-model score functions evaluated by an 8-lane group.
//
// Each function restates one reference forward() (file:line cited, relative to
// /root/reference/) in the canonical arithmetic of DESIGN.md §3.  All 8 lanes of
// the group call it with the same row pointers and all return the same score.
// GROUPING (kge_grouping): TAIL combines (h,r) first, HEAD combines (r,t) first.
#pragma once
#include "kge_common.cuh"

namespace kge {

struct TripleRows {
  const float* h[8];  // head-side rows   (ent / ent_re, ent_map / ent_im, ... up to 8 octonion parts)
  const float* t[8];  // tail-side rows
  const float* r[8];  // relation-side rows (rel / rel_re, w / rel_map / rel_im / M_r / theta)
};

// Latency-bound kernels (a few hundred groups: training batch, query preparation, pair resolution) read a
// triple's rows in dependent phases — norm of h, norm of r, norm of t, score, gradients —, each starting with a
// cold miss.  Requesting every row of the triple up front (one prefetch per 128-byte line, lanes of the group
// interleaved) overlaps those misses; the phases then hit in L2.  Row widths: d floats (h / t side), dr (r side).
KGE_DEV void prefetch_row_lines(const float* row, int nfloats, int lane) {
  if (row == nullptr) return;
  const char* p = reinterpret_cast<const char*>(row);
  for (int off = lane * 128; off < nfloats * 4; off += 8 * 128)
    asm volatile("prefetch.global.L2 [%0];" ::"l"(p + off));
}
KGE_DEV void prefetch_triple_rows(const TripleRows& R, int d, int dr, int lane) {
  // slot 0 only: in every model these rows are exactly d (h / t side) and >= dr (r side) floats wide, so no
  // request leaves its row; the further slots differ per model (ANALOGY's are d/2 wide) and are left alone
  prefetch_row_lines(R.h[0], d, lane);
  prefetch_row_lines(R.t[0], d, lane);
  prefetch_row_lines(R.r[0], dr, lane);
}

// Row pointers of triple (h, r, t).  htab/ttab/rtab: the table sets the head-side,
// tail-side and relation-side rows are read from (they differ only in 1-vs-all
// sweeps over a row shard, where the candidate side is the local shard).
template <int MODEL>
KGE_DEV void resolve_rows(TripleRows& R, const ModelParams& P, const float* const* htab,
                          const float* const* ttab, const float* const* rtab, int64_t h, int64_t r,
                          int64_t t) {
  const size_t d = (size_t)P.d, dr = (size_t)P.dr;
  R.h[1] = R.t[1] = R.r[1] = R.r[2] = R.h[2] = R.t[2] = nullptr;
  if (MODEL == KGE_SLM || MODEL == KGE_NTN || MODEL == KGE_SME || MODEL == KGE_SME_BL || MODEL == KGE_CONVKB) {
    // only the embedding rows are per-triple; the dense parameters are read through P.tab[2..]
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * dr;
  } else if (MODEL == KGE_KG2E) {  // [ent_mu, ent_sigma, rel_mu, rel_sigma]
    R.h[0] = htab[0] + h * d; R.h[1] = htab[1] + h * d; R.t[0] = ttab[0] + t * d; R.t[1] = ttab[1] + t * d;
    R.r[0] = rtab[2] + r * d; R.r[1] = rtab[3] + r * d;
  } else if (MODEL == KGE_QUATE || MODEL == KGE_OCTONIONE) {
    constexpr int C = (MODEL == KGE_QUATE) ? 4 : 8;   // [ent_1..ent_C, rel_1..rel_C]
#pragma unroll
    for (int c = 0; c < C; ++c) { R.h[c] = htab[c] + h * d; R.t[c] = ttab[c] + t * d; R.r[c] = rtab[C + c] + r * d; }
  } else if (MODEL == KGE_ANALOGY) {
    // [ent, rel, ent_re, ent_im, rel_re, rel_im]; slot 0: full-width rows, 1/2: half-width re/im
    const size_t d2 = d / 2;
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d;
    R.h[1] = htab[2] + h * d2; R.h[2] = htab[3] + h * d2;
    R.t[1] = ttab[2] + t * d2; R.t[2] = ttab[3] + t * d2;
    R.r[1] = rtab[4] + r * d2; R.r[2] = rtab[5] + r * d2;
  } else if (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d;
  } else if (MODEL == KGE_TRANSM) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d;
    R.r[1] = rtab[2] + r;  // theta[r]
  } else if (MODEL == KGE_CP) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[2] + t * d; R.r[0] = rtab[1] + r * d;
  } else if (MODEL == KGE_TRANSH) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d;
    R.r[1] = rtab[2] + r * d;
  } else if (MODEL == KGE_TRANSD) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d;
    R.h[1] = htab[2] + h * d; R.t[1] = ttab[2] + t * d; R.r[1] = rtab[3] + r * d;
  } else if (MODEL == KGE_TRANSR) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * dr;
    R.r[1] = rtab[2] + r * d * dr;
  } else if (MODEL == KGE_ROTATE) {
    R.h[0] = htab[0] + h * d; R.h[1] = htab[1] + h * d;
    R.t[0] = ttab[0] + t * d; R.t[1] = ttab[1] + t * d;
    R.r[0] = rtab[2] + r * d;
  } else if (MODEL == KGE_COMPLEX) {
    R.h[0] = htab[0] + h * d; R.h[1] = htab[1] + h * d;
    R.t[0] = ttab[0] + t * d; R.t[1] = ttab[1] + t * d;
    R.r[0] = rtab[2] + r * d; R.r[1] = rtab[3] + r * d;
  } else if (MODEL == KGE_HOLE) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d;
  } else if (MODEL == KGE_RESCAL) {
    R.h[0] = htab[0] + h * d; R.t[0] = ttab[0] + t * d; R.r[0] = rtab[1] + r * d * d;
  } else if (MODEL == KGE_SIMPLE || MODEL == KGE_SIMPLE_IGNR) {
    // h1 = ent_head[h], t2 = ent_tail[h]; t1 = ent_tail[t], h2 = ent_head[t] (pointwise.py:514-519)
    R.h[0] = htab[0] + h * d; R.h[1] = htab[1] + h * d;
    R.t[0] = ttab[1] + t * d; R.t[1] = ttab[0] + t * d;
    R.r[0] = rtab[2] + r * d; R.r[1] = rtab[3] + r * d;
  }
}

// RotatE query-side product (canonical): x o r = (xr re - xi im, xr im + xi re), or with the
// conjugate rotation x o conj(r) = (xr re + xi im, xi re - xr im)
KGE_DEV void rot_query(float xr, float xi, float re, float im, bool conj, float& qr, float& qi) {
  if (!conj) {
    qr = ffma(xr, re, -fmul(xi, im));
    qi = ffma(xr, im, fmul(xi, re));
  } else {
    qr = ffma(xr, re, fmul(xi, im));
    qi = ffma(xi, re, -fmul(xr, im));
  }
}

// group-scoped barrier for shared-memory scratch shared by the 8 lanes of a group
KGE_DEV void group_sync() { __syncwarp(group_mask()); }

// even part of a row: (x[j] + x[(d-j)%d]) / 2 for the 4 elements of chunk c (zero beyond d)
KGE_DEV float4 even_chunk(const float* __restrict__ row, int c, int d) {
  float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const int j = 4 * c + e;
    if (j < d) {
      const int jm = (j == 0) ? 0 : d - j;
      f4_at(o, e) = fmul(0.5f, fadd(__ldg(row + j), __ldg(row + jm)));
    }
  }
  return o;
}

// HoLE query-side vector  g[a] = sum_b qe[b] * rn[(a+b)%d]  (sequential b) for the lane's chunks;
// qe / rn / g live in the group's shared scratch (each d_pad floats).  pairwise.py:1119-1125 as
// written for torch<1.7, re-associated (see oracle/kge_oracle.c KGE_HOLE).
KGE_DEV void hole_query_vector(const float* qe, const float* rn, float* g, int d, int nch, int lane) {
  for (int c = lane; c < nch; c += 8) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int a = 4 * c + e;
      if (a < d) {
        float s = 0.f;
        int idx = a;
        for (int b = 0; b < d; ++b) {
          s = ffma(qe[b], rn[idx], s);
          idx = (idx + 1 == d) ? 0 : idx + 1;
        }
        f4_at(acc, e) = s;
      }
    }
    *reinterpret_cast<float4*>(g + 4 * c) = acc;
  }
}

// Hamilton product (QuatE/OctonionE._qmult, pointwise.py:962-968) in the canonical fma order
KGE_DEV void hyper_qmult(const float* A, const float* B, float* O) {
  O[0] = ffma(-A[3], B[3], ffma(-A[2], B[2], ffma(-A[1], B[1], fmul(A[0], B[0]))));
  O[1] = ffma(-B[2], A[3], ffma(A[2], B[3], ffma(B[0], A[1], fmul(A[0], B[1]))));
  O[2] = ffma(-B[3], A[1], ffma(A[3], B[1], ffma(B[0], A[2], fmul(A[0], B[2]))));
  O[3] = ffma(-B[1], A[2], ffma(A[1], B[2], ffma(B[0], A[3], fmul(A[0], B[3]))));
}
// unit-modulus relation (_onorm / QuatE.forward :681-685) and the product h (x) r^ for C = 4 / 8 parts
template <int C>
KGE_DEV void hyper_product(const float* hc, float* rc /* in: raw, out: normalised */, float* o, float* inv_out) {
  float den2 = fmul(rc[0], rc[0]);
#pragma unroll
  for (int c = 1; c < C; ++c) den2 = ffma(rc[c], rc[c], den2);
  const float inv = __frcp_rn(__fsqrt_rn(den2));
#pragma unroll
  for (int c = 0; c < C; ++c) rc[c] = fmul(rc[c], inv);
  if (inv_out) *inv_out = inv;
  if (C == 4) {
    hyper_qmult(hc, rc, o);
  } else {
    const float dstar[4] = {rc[4], -rc[5], -rc[6], -rc[7]}, cstar[4] = {rc[0], -rc[1], -rc[2], -rc[3]};
    float p1[4], p2[4], p3[4], p4[4];
    hyper_qmult(hc, rc, p1);
    hyper_qmult(dstar, hc + 4, p2);
    hyper_qmult(rc + 4, hc, p3);
    hyper_qmult(hc + 4, cstar, p4);
#pragma unroll
    for (int c = 0; c < 4; ++c) { o[c] = fsub(p1[c], p2[c]); o[4 + c] = fadd(p3[c], p4[c]); }
  }
}

// Shared tail of TransE/H/D/R/M forward(): L2-normalise h', r', t' and return
// ||h^ + r^ - t^||_p  (pairwise.py:69-76, :146-153, :266-273, :463-470).
// fh/fr/ft(c) return chunk c (4 elements, zero beyond the width) of each operand.
// CH > 0: the lane's chunks (c = lane + 8k, k < CH) are fetched ONCE into registers (load_trans_chunks) and
// both passes (norms, then distance) run from registers (trans_distance_regs) — one trip to memory instead of two.
template <int GROUPING>
KGE_DEV void trans_distance_step(const float4& a, const float4& b, const float4& cc, float ih, float ir, float it,
                                 int l1, float& acc) {
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    const float hn = fmul(f4_get(a, e), ih), rn = fmul(f4_get(b, e), ir), tn = fmul(f4_get(cc, e), it);
    float x;
    if (GROUPING == KGE_GROUP_TAIL) x = fsub(fadd(hn, rn), tn);
    else x = fadd(hn, fsub(rn, tn));
    if (l1) acc = fadd(acc, fabsf(x)); else acc = ffma(x, x, acc);
  }
}

template <int CH, class FH, class FR, class FT>
KGE_DEV void load_trans_chunks(FH fh, FR fr, FT ft, int nch, int lane, float4 (&A)[CH], float4 (&B)[CH],
                               float4 (&C)[CH]) {
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    const int c = lane + 8 * k;
    if (c < nch) { A[k] = fh(c); B[k] = fr(c); C[k] = ft(c); }
    else { A[k] = B[k] = C[k] = make_float4(0.f, 0.f, 0.f, 0.f); }
  }
}

template <int GROUPING, int CH>
KGE_DEV float trans_distance_regs(const float4 (&A)[CH], const float4 (&B)[CH], const float4 (&C)[CH], int l1) {
  float sh = 0.f, sr = 0.f, st = 0.f;
#pragma unroll
  for (int k = 0; k < CH; ++k) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sh = ffma(f4_get(A[k], e), f4_get(A[k], e), sh);
      sr = ffma(f4_get(B[k], e), f4_get(B[k], e), sr);
      st = ffma(f4_get(C[k], e), f4_get(C[k], e), st);
    }
  }
  const float ih = inv_norm_from_sumsq(group_sum(sh));
  const float ir = inv_norm_from_sumsq(group_sum(sr));
  const float it = inv_norm_from_sumsq(group_sum(st));
  float acc = 0.f;
  // zero-filled slots beyond the row add exact zeros: same bits as skipping them
#pragma unroll
  for (int k = 0; k < CH; ++k) trans_distance_step<GROUPING>(A[k], B[k], C[k], ih, ir, it, l1, acc);
  acc = group_sum(acc);
  return l1 ? acc : __fsqrt_rn(acc);
}

template <int GROUPING, int CH, class FH, class FR, class FT>
KGE_DEV float trans_distance_impl(FH fh, FR fr, FT ft, int nch, int lane, int l1) {
  if (CH > 0) {
    constexpr int K = CH > 0 ? CH : 1;
    float4 A[K], B[K], C[K];
    load_trans_chunks<K>(fh, fr, ft, nch, lane, A, B, C);
    return trans_distance_regs<GROUPING, K>(A, B, C, l1);
  }
  float sh = 0.f, sr = 0.f, st = 0.f;
#pragma unroll 2
  for (int c = lane; c < nch; c += 8) {
    const float4 a = fh(c), b = fr(c), cc = ft(c);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sh = ffma(f4_get(a, e), f4_get(a, e), sh);
      sr = ffma(f4_get(b, e), f4_get(b, e), sr);
      st = ffma(f4_get(cc, e), f4_get(cc, e), st);
    }
  }
  const float ih = inv_norm_from_sumsq(group_sum(sh));
  const float ir = inv_norm_from_sumsq(group_sum(sr));
  const float it = inv_norm_from_sumsq(group_sum(st));
  float acc = 0.f;
#pragma unroll 2
  for (int c = lane; c < nch; c += 8) trans_distance_step<GROUPING>(fh(c), fr(c), ft(c), ih, ir, it, l1, acc);
  acc = group_sum(acc);
  return l1 ? acc : __fsqrt_rn(acc);
}

// CHSEL >= 0: the register-cache depth is fixed at compile time (kernels whose host launcher
// picks it from d, so that narrow models keep a small register footprint / high occupancy);
// CHSEL < 0: chosen at run time.
template <int GROUPING, int CHSEL = -1, class FH, class FR, class FT>
KGE_DEV float trans_distance(FH fh, FR fr, FT ft, int nch, int lane, int l1) {
  if (CHSEL >= 0) return trans_distance_impl<GROUPING, (CHSEL >= 0 ? CHSEL : 0)>(fh, fr, ft, nch, lane, l1);
  if (nch <= 16) return trans_distance_impl<GROUPING, 2>(fh, fr, ft, nch, lane, l1);   // d <= 64
  if (nch <= 32) return trans_distance_impl<GROUPING, 4>(fh, fr, ft, nch, lane, l1);   // d <= 128
  if (nch <= 64) return trans_distance_impl<GROUPING, 8>(fh, fr, ft, nch, lane, l1);   // d <= 256
  return trans_distance_impl<GROUPING, 0>(fh, fr, ft, nch, lane, l1);
}

template <int VEC>
KGE_DEV float group_dot(const float* __restrict__ a, const float* __restrict__ b, int d, int nch, int lane) {
  float s = 0.f;
#pragma unroll 2
  for (int c = lane; c < nch; c += 8) {
    const float4 x = ld_chunk<VEC>(a, c, d), y = ld_chunk<VEC>(b, c, d);
#pragma unroll
    for (int e = 0; e < 4; ++e) s = ffma(f4_get(x, e), f4_get(y, e), s);
  }
  return group_sum(s);
}

// ---- dense-layer models (SLM / NTN / SME / SME_BL): shared forward pieces left in the group's scratch
struct DenseCtx {
  float ih, it, ir;                 // inverse norms
  bool clamp_h, clamp_t, clamp_r;   // norm below eps (F.normalize divides by the constant eps)
  float *hn, *tn, *rn;              // normalised operands
  float *act, *A, *B;               // SLM/NTN: tanh(pre), (h^ mr1), (t^ mr2)
  float *gu, *gv, *u1, *u2, *v1, *v2;  // SME / SME_BL
};
inline __host__ __device__ int dense_dm(int d, int K) { return ((d > K ? d : K) + 3) / 4 * 4; }

template <int VEC>
KGE_DEV void dense_normalise(const TripleRows& R, int d, int K, int lane, DenseCtx& X) {
  const int nch = (d + 3) >> 2, nchk = (K + 3) >> 2;
  float sh = 0.f, st = 0.f, sr = 0.f;
  for (int c = lane; c < nch; c += 8) {
    const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
    for (int e = 0; e < 4; ++e) { sh = ffma(f4_get(a, e), f4_get(a, e), sh); st = ffma(f4_get(b, e), f4_get(b, e), st); }
  }
  for (int c = lane; c < nchk; c += 8) {
    const float4 b = ld_chunk<VEC>(R.r[0], c, K);
#pragma unroll
    for (int e = 0; e < 4; ++e) sr = ffma(f4_get(b, e), f4_get(b, e), sr);
  }
  sh = group_sum(sh); st = group_sum(st); sr = group_sum(sr);
  X.ih = inv_norm_from_sumsq(sh); X.it = inv_norm_from_sumsq(st); X.ir = inv_norm_from_sumsq(sr);
  X.clamp_h = __fsqrt_rn(sh) < 1e-12f; X.clamp_t = __fsqrt_rn(st) < 1e-12f; X.clamp_r = __fsqrt_rn(sr) < 1e-12f;
  for (int c = lane; c < nch; c += 8) {
    const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.t[0], c, d);
    *reinterpret_cast<float4*>(X.hn + 4 * c) = make_float4(fmul(a.x, X.ih), fmul(a.y, X.ih), fmul(a.z, X.ih), fmul(a.w, X.ih));
    *reinterpret_cast<float4*>(X.tn + 4 * c) = make_float4(fmul(b.x, X.it), fmul(b.y, X.it), fmul(b.z, X.it), fmul(b.w, X.it));
  }
  for (int c = lane; c < nchk; c += 8) {
    const float4 b = ld_chunk<VEC>(R.r[0], c, K);
    *reinterpret_cast<float4*>(X.rn + 4 * c) = make_float4(fmul(b.x, X.ir), fmul(b.y, X.ir), fmul(b.z, X.ir), fmul(b.w, X.ir));
  }
  group_sync();
}

// scratch layout (dm floats each): hn, tn, rn, act, A, B
template <int MODEL, int VEC>
KGE_DEV void slm_ntn_fill(const TripleRows& R, const ModelParams& P, int lane, float* scratch, DenseCtx& X) {
  const int d = P.d, K = P.dr, nch = (d + 3) >> 2, nchk = (K + 3) >> 2, dm = dense_dm(d, K);
  X.hn = scratch; X.tn = scratch + dm; X.rn = scratch + 2 * dm; X.act = scratch + 3 * dm;
  X.A = scratch + 4 * dm; X.B = scratch + 5 * dm;
  dense_normalise<VEC>(R, d, K, lane, X);
  const float* mr1 = P.tab[2];
  const float* mr2 = P.tab[3];
  for (int c = lane; c < nchk; c += 8) {
    float4 a = make_float4(0.f, 0.f, 0.f, 0.f), b = a;
    for (int i = 0; i < d; ++i) {
      const float hi = X.hn[i], ti = X.tn[i];
      const float4 m1 = ld_chunk<VEC>(mr1 + (size_t)i * K, c, K), m2 = ld_chunk<VEC>(mr2 + (size_t)i * K, c, K);
#pragma unroll
      for (int e = 0; e < 4; ++e) { f4_at(a, e) = ffma(hi, f4_get(m1, e), f4_get(a, e)); f4_at(b, e) = ffma(ti, f4_get(m2, e), f4_get(b, e)); }
    }
    if (MODEL == KGE_SLM) {
      float4 o;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(o, e) = tanh_canon(fadd(f4_get(a, e), f4_get(b, e)));
      *reinterpret_cast<float4*>(X.act + 4 * c) = o;
    } else {
      *reinterpret_cast<float4*>(X.A + 4 * c) = a;
      *reinterpret_cast<float4*>(X.B + 4 * c) = b;
    }
  }
  if (MODEL == KGE_NTN) {
    group_sync();
    const float* br = P.tab[4];
    for (int k = 0; k < K; ++k) {
      const float* W = P.tab[5] + (size_t)k * d * d;
      float part = 0.f;
      for (int c = lane; c < nch; c += 8) {
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int i = 0; i < d; ++i) {
          const float hi = X.hn[i];
          const float4 w = ld_chunk<VEC>(W + (size_t)i * d, c, d);
#pragma unroll
          for (int e = 0; e < 4; ++e) f4_at(v, e) = ffma(hi, f4_get(w, e), f4_get(v, e));
        }
        const float4 tt = *reinterpret_cast<const float4*>(X.tn + 4 * c);
#pragma unroll
        for (int e = 0; e < 4; ++e) part = ffma(f4_get(v, e), f4_get(tt, e), part);
      }
      const float bil = group_sum(part);
      if (lane == 0) X.act[k] = tanh_canon(fadd(fadd(fadd(bil, X.A[k]), X.B[k]), __ldg(br + k)));
    }
    if (lane == 0) for (int k = K; k < nchk * 4; ++k) X.act[k] = 0.f;
  }
  group_sync();
}

// scratch layout (dm floats each): hn, rn, tn, gu, gv, u1, u2, v1, v2
template <int MODEL, int VEC>
KGE_DEV void sme_fill(const TripleRows& R, const ModelParams& P, int lane, float* scratch, DenseCtx& X) {
  const int d = P.d, nch = (d + 3) >> 2, dm = nch * 4;
  X.hn = scratch; X.rn = scratch + dm; X.tn = scratch + 2 * dm; X.gu = scratch + 3 * dm; X.gv = scratch + 4 * dm;
  X.u1 = scratch + 5 * dm; X.u2 = scratch + 6 * dm; X.v1 = scratch + 7 * dm; X.v2 = scratch + 8 * dm;
  dense_normalise<VEC>(R, d, d, lane, X);
  const float *mu1 = P.tab[2], *mu2 = P.tab[3], *bu = P.tab[4], *mv1 = P.tab[5], *mv2 = P.tab[6], *bv = P.tab[7];
  for (int c = lane; c < nch; c += 8) {
    float4 GU = make_float4(0.f, 0.f, 0.f, 0.f), GV = GU, U1 = GU, U2 = GU, V1 = GU, V2 = GU;
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const int k = 4 * c + e;
      if (k < d) {
        float u1 = 0.f, u2 = 0.f, v1 = 0.f, v2 = 0.f;
        const float *r1 = mu1 + (size_t)k * d, *r2 = mu2 + (size_t)k * d, *r3 = mv1 + (size_t)k * d, *r4 = mv2 + (size_t)k * d;
        for (int i = 0; i < d; ++i) {
          const float hi = X.hn[i], ri = X.rn[i], ti = X.tn[i];
          u1 = ffma(__ldg(r1 + i), hi, u1); u2 = ffma(__ldg(r2 + i), ri, u2);
          v1 = ffma(__ldg(r3 + i), ti, v1); v2 = ffma(__ldg(r4 + i), ri, v2);
        }
        f4_at(U1, e) = u1; f4_at(U2, e) = u2; f4_at(V1, e) = v1; f4_at(V2, e) = v2;
        if (MODEL == KGE_SME) { f4_at(GU, e) = fadd(fadd(u1, u2), __ldg(bu + k)); f4_at(GV, e) = fadd(fadd(v1, v2), __ldg(bv + k)); }
        else { f4_at(GU, e) = fadd(fmul(u1, u2), __ldg(bu + k)); f4_at(GV, e) = fadd(fmul(v1, v2), __ldg(bv + k)); }
      }
    }
    *reinterpret_cast<float4*>(X.gu + 4 * c) = GU; *reinterpret_cast<float4*>(X.gv + 4 * c) = GV;
    *reinterpret_cast<float4*>(X.u1 + 4 * c) = U1; *reinterpret_cast<float4*>(X.u2 + 4 * c) = U2;
    *reinterpret_cast<float4*>(X.v1 + 4 * c) = V1; *reinterpret_cast<float4*>(X.v2 + 4 * c) = V2;
  }
  group_sync();
}

// `scratch`: per-group shared memory, only used by TransR (2 * dr_pad floats).
template <int MODEL, int VEC, int GROUPING, int CHSEL = -1>
KGE_DEV float score_group(const TripleRows& R, const ModelParams& P, int lane, float* scratch) {
  const int d = P.d;
  const int nch = (d + 3) >> 2;
  if (MODEL == KGE_TRANSE || MODEL == KGE_TRANSM) {
    // TransE.forward pairwise.py:56-93; TransM.forward pairwise.py:325-347
    const float dist = trans_distance<GROUPING, CHSEL>(
        [&](int c) { return ld_chunk<VEC>(R.h[0], c, d); },
        [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); },
        [&](int c) { return ld_chunk<VEC>(R.t[0], c, d); }, nch, lane, P.l1);
    if (MODEL == KGE_TRANSM) return fmul(__ldg(R.r[1]), dist);
    return dist;
  } else if (MODEL == KGE_TRANSH) {
    // TransH.embed/_projection pairwise.py:166-182: e_perp = e - (e . w~) w~
    float sw = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 w = ld_chunk<VEC>(R.r[1], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) sw = ffma(f4_get(w, e), f4_get(w, e), sw);
    }
    const float iw = inv_norm_from_sumsq(group_sum(sw));
    float ah = 0.f, at = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 w = ld_chunk<VEC>(R.r[1], c, d), a = ld_chunk<VEC>(R.h[0], c, d),
                   b = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float wn = fmul(f4_get(w, e), iw);
        ah = ffma(f4_get(a, e), wn, ah);
        at = ffma(f4_get(b, e), wn, at);
      }
    }
    ah = group_sum(ah); at = group_sum(at);
    auto proj = [&](const float* row, float a, int c) {
      const float4 w = ld_chunk<VEC>(R.r[1], c, d), x = ld_chunk<VEC>(row, c, d);
      float4 o;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(o, e) = ffma(-a, fmul(f4_get(w, e), iw), f4_get(x, e));
      return o;
    };
    return trans_distance<GROUPING, CHSEL>([&](int c) { return proj(R.h[0], ah, c); },
                                    [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); },
                                    [&](int c) { return proj(R.t[0], at, c); }, nch, lane, P.l1);
  } else if (MODEL == KGE_TRANSD) {
    // TransD.embed/_projection pairwise.py:240-249,275-278: e' = e + (e . e_m) r_m
    const float ah = group_dot<VEC>(R.h[0], R.h[1], d, nch, lane);
    const float at = group_dot<VEC>(R.t[0], R.t[1], d, nch, lane);
    auto proj = [&](const float* row, float a, int c) {
      const float4 rm = ld_chunk<VEC>(R.r[1], c, d), x = ld_chunk<VEC>(row, c, d);
      float4 o;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(o, e) = ffma(a, f4_get(rm, e), f4_get(x, e));
      return o;
    };
    return trans_distance<GROUPING, CHSEL>([&](int c) { return proj(R.h[0], ah, c); },
                                    [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); },
                                    [&](int c) { return proj(R.t[0], at, c); }, nch, lane, P.l1);
  } else if (MODEL == KGE_TRANSR) {
    // TransR.embed/transform pairwise.py:405-442 then forward :463-470
    const int dr = P.dr, nchr = (dr + 3) >> 2, drp = nchr * 4;
    float sh = 0.f, st = 0.f, sr = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) { sh = ffma(f4_get(a, e), f4_get(a, e), sh); st = ffma(f4_get(b, e), f4_get(b, e), st); }
    }
    for (int c = lane; c < nchr; c += 8) {
      const float4 b = ld_chunk<VEC>(R.r[0], c, dr);
#pragma unroll
      for (int e = 0; e < 4; ++e) sr = ffma(f4_get(b, e), f4_get(b, e), sr);
    }
    const float ih = inv_norm_from_sumsq(group_sum(sh));
    const float it = inv_norm_from_sumsq(group_sum(st));
    const float ir = inv_norm_from_sumsq(group_sum(sr));
    float* hp = scratch;        // [drp]
    float* tp = scratch + drp;  // [drp]
    // h'_k = sum_j h^_j M[j,k], sequential in j (single accumulator per output element);
    // lane l owns the output chunks c = l, l+8, ...
    for (int c = lane; c < nchr; c += 8) {
      float4 ah = make_float4(0.f, 0.f, 0.f, 0.f), at = ah;
      for (int j = 0; j < d; ++j) {
        const float hn = fmul(__ldg(R.h[0] + j), ih), tn = fmul(__ldg(R.t[0] + j), it);
        const float4 mrow = ld_chunk<VEC>(R.r[1] + (size_t)j * dr, c, dr);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          f4_at(ah, e) = ffma(hn, f4_get(mrow, e), f4_get(ah, e));
          f4_at(at, e) = ffma(tn, f4_get(mrow, e), f4_get(at, e));
        }
      }
      *reinterpret_cast<float4*>(hp + 4 * c) = ah;
      *reinterpret_cast<float4*>(tp + 4 * c) = at;
    }
    group_sync();   // this group's lanes only: callers branch per group (train_hinge_kernel: active pairs)
    return trans_distance<GROUPING, CHSEL>(
        [&](int c) { return *reinterpret_cast<const float4*>(hp + 4 * c); },
        [&](int c) {
          const float4 b = ld_chunk<VEC>(R.r[0], c, dr);
          return make_float4(fmul(b.x, ir), fmul(b.y, ir), fmul(b.z, ir), fmul(b.w, ir));
        },
        [&](int c) { return *reinterpret_cast<const float4*>(tp + 4 * c); }, nchr, lane, P.l1);
  } else if (MODEL == KGE_ROTATE) {
    // RotatE.embed/forward pairwise.py:765-791.  TAIL: |h o r - t|^2 as written; HEAD: the query
    // side is t o conj(r) and the candidate h stays raw: |t o conj(r) - h|^2 (equal for the unit
    // rotation e^{i theta}; rule 5: each grouping has its own canonical arithmetic)
    float acc = 0.f;
#pragma unroll 2
    for (int c = lane; c < nch; c += 8) {
      const float4 hr = ld_chunk<VEC>(R.h[0], c, d), hi = ld_chunk<VEC>(R.h[1], c, d),
                   rr = ld_chunk<VEC>(R.r[0], c, d), tr = ld_chunk<VEC>(R.t[0], c, d),
                   ti = ld_chunk<VEC>(R.t[1], c, d);
      float4 sr4, si4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float im, re, qr, qi;
        sincos_canon(fmul(f4_get(rr, e), P.phase), im, re);
        if (GROUPING == KGE_GROUP_TAIL) {
          rot_query(f4_get(hr, e), f4_get(hi, e), re, im, false, qr, qi);
          f4_at(sr4, e) = fsub(qr, f4_get(tr, e));
          f4_at(si4, e) = fsub(qi, f4_get(ti, e));
        } else {
          rot_query(f4_get(tr, e), f4_get(ti, e), re, im, true, qr, qi);
          f4_at(sr4, e) = fsub(qr, f4_get(hr, e));
          f4_at(si4, e) = fsub(qi, f4_get(hi, e));
        }
      }
      // two-term sums accumulate chunk-wise: the chunk's 4 first terms, then its 4 second terms
      // (DESIGN.md §3 rule 6)
#pragma unroll
      for (int e = 0; e < 4; ++e) acc = ffma(f4_get(sr4, e), f4_get(sr4, e), acc);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc = ffma(f4_get(si4, e), f4_get(si4, e), acc);
    }
    return fsub(group_sum(acc), P.margin);
  } else if (MODEL == KGE_DISTMULT || MODEL == KGE_CP) {
    // DistMult.forward pointwise.py:444-446; CP.forward pointwise.py:374-376
    float acc = 0.f;
#pragma unroll 2
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.r[0], c, d),
                   cc = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (GROUPING == KGE_GROUP_TAIL) acc = ffma(fmul(f4_get(a, e), f4_get(b, e)), f4_get(cc, e), acc);
        else acc = ffma(f4_get(a, e), fmul(f4_get(b, e), f4_get(cc, e)), acc);
      }
    }
    return -group_sum(acc);
  } else if (MODEL == KGE_CONVKB) {
    // ConvKB.forward pointwise.py:302-318 in its collapsed affine form (include/kge_b200.h):
    // three canonical sums, combined in the grouping's order, plus the constant
    const float* A = P.tab[2];
    float sh = 0.f, sr = 0.f, st = 0.f;
#pragma unroll 2
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.r[0], c, d), cc = ld_chunk<VEC>(R.t[0], c, d);
      const float4 wa = ld_chunk<VEC>(A, c, d), wb = ld_chunk<VEC>(A + d, c, d), wc = ld_chunk<VEC>(A + 2 * (size_t)d, c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        sh = ffma(f4_get(a, e), f4_get(wa, e), sh);
        sr = ffma(f4_get(b, e), f4_get(wb, e), sr);
        st = ffma(f4_get(cc, e), f4_get(wc, e), st);
      }
    }
    sh = group_sum(sh); sr = group_sum(sr); st = group_sum(st);
    const float s = (GROUPING == KGE_GROUP_TAIL) ? fadd(fadd(sh, sr), st) : fadd(sh, fadd(sr, st));
    return fadd(s, __ldg(P.tab[3]));
  } else if (MODEL == KGE_COMPLEX) {
    // Complex.forward pointwise.py:163-188
    float acc = 0.f;
#pragma unroll 2
    for (int c = lane; c < nch; c += 8) {
      const float4 hr = ld_chunk<VEC>(R.h[0], c, d), hi = ld_chunk<VEC>(R.h[1], c, d),
                   rr = ld_chunk<VEC>(R.r[0], c, d), ri = ld_chunk<VEC>(R.r[1], c, d),
                   tr = ld_chunk<VEC>(R.t[0], c, d), ti = ld_chunk<VEC>(R.t[1], c, d);
      float4 qr4, qi4;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (GROUPING == KGE_GROUP_TAIL) {
          f4_at(qr4, e) = ffma(f4_get(hr, e), f4_get(rr, e), -fmul(f4_get(hi, e), f4_get(ri, e)));
          f4_at(qi4, e) = ffma(f4_get(hi, e), f4_get(rr, e), fmul(f4_get(hr, e), f4_get(ri, e)));
        } else {
          f4_at(qr4, e) = ffma(f4_get(tr, e), f4_get(rr, e), fmul(f4_get(ti, e), f4_get(ri, e)));
          f4_at(qi4, e) = ffma(f4_get(ti, e), f4_get(rr, e), -fmul(f4_get(tr, e), f4_get(ri, e)));
        }
      }
      // chunk-wise: 4 real-part terms, then 4 imaginary-part terms (DESIGN.md §3 rule 6)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        acc = (GROUPING == KGE_GROUP_TAIL) ? ffma(f4_get(qr4, e), f4_get(tr, e), acc) : ffma(f4_get(hr, e), f4_get(qr4, e), acc);
#pragma unroll
      for (int e = 0; e < 4; ++e)
        acc = (GROUPING == KGE_GROUP_TAIL) ? ffma(f4_get(qi4, e), f4_get(ti, e), acc) : ffma(f4_get(hi, e), f4_get(qi4, e), acc);
    }
    return -group_sum(acc);
  } else if (MODEL == KGE_SLM || MODEL == KGE_NTN) {
    // SLM.forward/layer pairwise.py:525-541; NTN.forward/train_layer pairwise.py:919-960
    const int K = P.dr, nchk = (K + 3) >> 2;
    DenseCtx X;
    slm_ntn_fill<MODEL, VEC>(R, P, lane, scratch, X);
    float acc = 0.f;
    for (int c = lane; c < nchk; c += 8) {
      const float4 rr = *reinterpret_cast<const float4*>(X.rn + 4 * c), aa = *reinterpret_cast<const float4*>(X.act + 4 * c);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc = ffma(f4_get(rr, e), f4_get(aa, e), acc);
    }
    group_sync();
    return -group_sum(acc);
  } else if (MODEL == KGE_SME || MODEL == KGE_SME_BL) {
    // SME.forward pairwise.py:617-661 / SME_BL.forward :680-724
    DenseCtx X;
    sme_fill<MODEL, VEC>(R, P, lane, scratch, X);
    float acc = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 gu = *reinterpret_cast<const float4*>(X.gu + 4 * c), gv = *reinterpret_cast<const float4*>(X.gv + 4 * c);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc = ffma(f4_get(gu, e), f4_get(gv, e), acc);
    }
    group_sync();
    const float tot = group_sum(acc);
    return MODEL == KGE_SME ? -tot : tot;
  } else if (MODEL == KGE_KG2E) {
    // KG2E.forward / _cal_score_kl_divergence pairwise.py:1021-1084 (grouping-independent)
    const float* rows6[6] = {R.h[0], R.h[1], R.r[0], R.r[1], R.t[0], R.t[1]};
    float inv[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      float s = 0.f;
      for (int c = lane; c < nch; c += 8) {
        const float4 x = ld_chunk<VEC>(rows6[k], c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) s = ffma(f4_get(x, e), f4_get(x, e), s);
      }
      inv[k] = __frcp_rn(__fsqrt_rn(group_sum(s)));
    }
    float T = 0.f, M = 0.f, D = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 hm = ld_chunk<VEC>(R.h[0], c, d), hs = ld_chunk<VEC>(R.h[1], c, d), rm = ld_chunk<VEC>(R.r[0], c, d),
                   rs = ld_chunk<VEC>(R.r[1], c, d), tm = ld_chunk<VEC>(R.t[0], c, d), ts = ld_chunk<VEC>(R.t[1], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (4 * c + e < d) {  // (padding would feed 0/0 into the divisions)
          const float cs = fadd(fmul(f4_get(hs, e), inv[1]), fmul(f4_get(rs, e), inv[3]));
          const float cm = fadd(fmul(f4_get(hm, e), inv[0]), fmul(f4_get(rm, e), inv[2]));
          const float st = fmul(f4_get(ts, e), inv[5]);
          const float x = fsub(fmul(f4_get(tm, e), inv[4]), cm);
          T = fadd(T, __fdiv_rn(cs, st));
          M = fadd(M, __fdiv_rn(fmul(x, x), st));
          D = fadd(D, fsub(log_canon(st), log_canon(cs)));
        }
      }
    }
    T = group_sum(T); M = group_sum(M); D = group_sum(D);
    return fsub(fadd(fadd(T, M), D), (float)d);
  } else if (MODEL == KGE_QUATE || MODEL == KGE_OCTONIONE) {
    // QuatE.forward pointwise.py:678-694 / OctonionE.forward :886-899 (grouping-independent)
    constexpr int C = (MODEL == KGE_QUATE) ? 4 : 8;
    float acc = 0.f;
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        if (j < d) {
          float hc[C], rc[C], tc[C], o[C];
#pragma unroll
          for (int k = 0; k < C; ++k) { hc[k] = __ldg(R.h[k] + j); rc[k] = __ldg(R.r[k] + j); tc[k] = __ldg(R.t[k] + j); }
          hyper_product<C>(hc, rc, o, nullptr);
#pragma unroll
          for (int k = 0; k < C; ++k) acc = ffma(o[k], tc[k], acc);
        }
      }
    }
    return -group_sum(acc);
  } else if (MODEL == KGE_ANALOGY) {
    // ANALOGY.forward pointwise.py:97-104: ComplEx(d/2) + DistMult(d)
    const int d2 = d / 2, nch2 = (d2 + 3) >> 2;
    float ac = 0.f;
    for (int c = lane; c < nch2; c += 8) {
      const float4 hr = ld_chunk<VEC>(R.h[1], c, d2), hi = ld_chunk<VEC>(R.h[2], c, d2),
                   rr = ld_chunk<VEC>(R.r[1], c, d2), ri = ld_chunk<VEC>(R.r[2], c, d2),
                   tr = ld_chunk<VEC>(R.t[1], c, d2), ti = ld_chunk<VEC>(R.t[2], c, d2);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (GROUPING == KGE_GROUP_TAIL) {
          const float qr = ffma(f4_get(hr, e), f4_get(rr, e), -fmul(f4_get(hi, e), f4_get(ri, e)));
          const float qi = ffma(f4_get(hi, e), f4_get(rr, e), fmul(f4_get(hr, e), f4_get(ri, e)));
          ac = ffma(qr, f4_get(tr, e), ac);
          ac = ffma(qi, f4_get(ti, e), ac);
        } else {
          const float qr = ffma(f4_get(tr, e), f4_get(rr, e), fmul(f4_get(ti, e), f4_get(ri, e)));
          const float qi = ffma(f4_get(ti, e), f4_get(rr, e), -fmul(f4_get(tr, e), f4_get(ri, e)));
          ac = ffma(f4_get(hr, e), qr, ac);
          ac = ffma(f4_get(hi, e), qi, ac);
        }
      }
    }
    float ad = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.r[0], c, d), cc = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (GROUPING == KGE_GROUP_TAIL) ad = ffma(fmul(f4_get(a, e), f4_get(b, e)), f4_get(cc, e), ad);
        else ad = ffma(f4_get(a, e), fmul(f4_get(b, e), f4_get(cc, e)), ad);
      }
    }
    return fsub(-group_sum(ac), group_sum(ad));
  } else if (MODEL == KGE_HOLE) {
    // scratch: rn[dp], qe[dp], g[dp]
    const int dp = nch * 4;
    float *rn = scratch, *qe = scratch + dp, *g = scratch + 2 * dp;
    float sr = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 b = ld_chunk<VEC>(R.r[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) sr = ffma(f4_get(b, e), f4_get(b, e), sr);
    }
    const float ir = inv_norm_from_sumsq(group_sum(sr));
    const float* qrow = (GROUPING == KGE_GROUP_TAIL) ? R.h[0] : R.t[0];
    const float* crow = (GROUPING == KGE_GROUP_TAIL) ? R.t[0] : R.h[0];
    for (int c = lane; c < nch; c += 8) {
      const float4 b = ld_chunk<VEC>(R.r[0], c, d);
      *reinterpret_cast<float4*>(rn + 4 * c) = make_float4(fmul(b.x, ir), fmul(b.y, ir), fmul(b.z, ir), fmul(b.w, ir));
      *reinterpret_cast<float4*>(qe + 4 * c) = even_chunk(qrow, c, d);
    }
    group_sync();
    hole_query_vector(qe, rn, g, d, nch, lane);
    float acc = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 gv = *reinterpret_cast<const float4*>(g + 4 * c);
      const float4 ce = even_chunk(crow, c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc = ffma(f4_get(gv, e), f4_get(ce, e), acc);
    }
    group_sync();  // scratch may be reused by the caller's next evaluation
    return -sigmoid_canon(group_sum(acc));
  } else if (MODEL == KGE_RESCAL) {
    // scratch: v[dp].  TAIL: v = h^T M (sequential j), s = RSUM v.t ; HEAD: u = M t (sequential k), s = RSUM h.u
    const float* M = R.r[0];
    float* v = scratch;
    if (GROUPING == KGE_GROUP_TAIL) {
      for (int c = lane; c < nch; c += 8) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int j = 0; j < d; ++j) {
          const float hj = __ldg(R.h[0] + j);
          const float4 mrow = ld_chunk<VEC>(M + (size_t)j * d, c, d);
#pragma unroll
          for (int e = 0; e < 4; ++e) f4_at(a, e) = ffma(hj, f4_get(mrow, e), f4_get(a, e));
        }
        *reinterpret_cast<float4*>(v + 4 * c) = a;
      }
    } else {
      for (int c = lane; c < nch; c += 8) {
        float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
        for (int kc = 0; kc < nch; ++kc) {
          const float4 tv = ld_chunk<VEC>(R.t[0], kc, d);
#pragma unroll
          for (int e = 0; e < 4; ++e) {
            const int j = 4 * c + e;
            if (j < d) {
              const float4 mrow = ld_chunk<VEC>(M + (size_t)j * d, kc, d);
#pragma unroll
              for (int q = 0; q < 4; ++q) f4_at(a, e) = ffma(f4_get(mrow, q), f4_get(tv, q), f4_get(a, e));
            }
          }
        }
        *reinterpret_cast<float4*>(v + 4 * c) = a;
      }
    }
    const float* other = (GROUPING == KGE_GROUP_TAIL) ? R.t[0] : R.h[0];
    float acc = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = *reinterpret_cast<const float4*>(v + 4 * c);
      const float4 o = ld_chunk<VEC>(other, c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) acc = ffma(f4_get(a, e), f4_get(o, e), acc);
    }
    return -group_sum(acc);
  } else if (MODEL == KGE_SIMPLE || MODEL == KGE_SIMPLE_IGNR) {
    // SimplE.forward pointwise.py:522-526 / SimplE_ignr.forward :573-581
    const float half = (MODEL == KGE_SIMPLE) ? 0.5f : 1.0f;
    float acc = 0.f;
#pragma unroll 2
    for (int c = lane; c < nch; c += 8) {
      const float4 h1 = ld_chunk<VEC>(R.h[0], c, d), t2 = ld_chunk<VEC>(R.h[1], c, d),
                   t1 = ld_chunk<VEC>(R.t[0], c, d), h2 = ld_chunk<VEC>(R.t[1], c, d),
                   r1 = ld_chunk<VEC>(R.r[0], c, d), r2 = ld_chunk<VEC>(R.r[1], c, d);
      float4 qa, qb;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        if (GROUPING == KGE_GROUP_TAIL) {
          f4_at(qa, e) = fmul(f4_get(h1, e), f4_get(r1, e));
          f4_at(qb, e) = fmul(fmul(f4_get(t2, e), f4_get(r2, e)), half);
        } else {
          f4_at(qa, e) = fmul(f4_get(r1, e), f4_get(t1, e));
          f4_at(qb, e) = fmul(fmul(f4_get(r2, e), f4_get(h2, e)), half);
        }
      }
      // chunk-wise: 4 terms of the first product, then 4 of the second (DESIGN.md §3 rule 6)
#pragma unroll
      for (int e = 0; e < 4; ++e)
        acc = (GROUPING == KGE_GROUP_TAIL) ? ffma(f4_get(qa, e), f4_get(t1, e), acc) : ffma(f4_get(h1, e), f4_get(qa, e), acc);
#pragma unroll
      for (int e = 0; e < 4; ++e)
        acc = (GROUPING == KGE_GROUP_TAIL) ? ffma(f4_get(qb, e), f4_get(h2, e), acc) : ffma(f4_get(t2, e), f4_get(qb, e), acc);
    }
    const float init = group_sum(acc);
    return -fminf(fmaxf(init, -20.0f), 20.0f);
  }
  return 0.f;
}

// register-cache depth for a distance model of width d (see trans_distance)
inline int ch_select(int width) {
  const int nch = (width + 3) >> 2;
  return nch <= 16 ? 2 : (nch <= 32 ? 4 : (nch <= 64 ? 8 : 0));
}
constexpr bool is_distance_model(int model) {
  return model == KGE_TRANSE || model == KGE_TRANSM || model == KGE_TRANSH || model == KGE_TRANSD ||
         model == KGE_TRANSR;
}

// shared-memory floats one 8-lane group needs (TransR only)
inline size_t group_scratch_floats(const kge_model_t* m) {
  const size_t dp = (size_t)(((m->dim + 3) >> 2) * 4);
  if (m->model == KGE_SLM || m->model == KGE_NTN) return 6 * (size_t)dense_dm(m->dim, m->rel_dim);
  if (m->model == KGE_SME || m->model == KGE_SME_BL) return 9 * dp;
  if (m->model == KGE_HOLE) return 3 * dp;
  if (m->model == KGE_RESCAL) return dp;
  if (m->model != KGE_TRANSR) return 0;
  return (size_t)2 * (size_t)(((m->rel_dim + 3) >> 2) * 4);
}

// Dispatch helper: calls F.template run<MODEL, VEC>() for the runtime (model, vec).
#define KGE_DISPATCH_MODEL_VEC(model, vec, CALL)                                   \
  do {                                                                             \
    switch (model) {                                                               \
      case KGE_TRANSE: KGE_DISPATCH_VEC(KGE_TRANSE, vec, CALL); break;             \
      case KGE_TRANSH: KGE_DISPATCH_VEC(KGE_TRANSH, vec, CALL); break;             \
      case KGE_TRANSD: KGE_DISPATCH_VEC(KGE_TRANSD, vec, CALL); break;             \
      case KGE_TRANSR: KGE_DISPATCH_VEC(KGE_TRANSR, vec, CALL); break;             \
      case KGE_ROTATE: KGE_DISPATCH_VEC(KGE_ROTATE, vec, CALL); break;             \
      case KGE_DISTMULT: KGE_DISPATCH_VEC(KGE_DISTMULT, vec, CALL); break;         \
      case KGE_COMPLEX: KGE_DISPATCH_VEC(KGE_COMPLEX, vec, CALL); break;           \
      case KGE_CP: KGE_DISPATCH_VEC(KGE_CP, vec, CALL); break;                     \
      case KGE_TRANSM: KGE_DISPATCH_VEC(KGE_TRANSM, vec, CALL); break;             \
      case KGE_HOLE: KGE_DISPATCH_VEC(KGE_HOLE, vec, CALL); break;                 \
      case KGE_ANALOGY: KGE_DISPATCH_VEC(KGE_ANALOGY, vec, CALL); break;           \
      case KGE_QUATE: KGE_DISPATCH_VEC(KGE_QUATE, vec, CALL); break;               \
      case KGE_KG2E: KGE_DISPATCH_VEC(KGE_KG2E, vec, CALL); break;                 \
      case KGE_SLM: KGE_DISPATCH_VEC(KGE_SLM, vec, CALL); break;                   \
      case KGE_NTN: KGE_DISPATCH_VEC(KGE_NTN, vec, CALL); break;                   \
      case KGE_SME: KGE_DISPATCH_VEC(KGE_SME, vec, CALL); break;                   \
      case KGE_SME_BL: KGE_DISPATCH_VEC(KGE_SME_BL, vec, CALL); break;             \
      case KGE_OCTONIONE: KGE_DISPATCH_VEC(KGE_OCTONIONE, vec, CALL); break;       \
      case KGE_RESCAL: KGE_DISPATCH_VEC(KGE_RESCAL, vec, CALL); break;             \
      case KGE_SIMPLE: KGE_DISPATCH_VEC(KGE_SIMPLE, vec, CALL); break;             \
      case KGE_SIMPLE_IGNR: KGE_DISPATCH_VEC(KGE_SIMPLE_IGNR, vec, CALL); break;   \
      case KGE_CONVKB: KGE_DISPATCH_VEC(KGE_CONVKB, vec, CALL); break;             \
      default: ::kge::set_error("model id %d not supported", (int)(model)); return KGE_ENOTSUP; \
    }                                                                              \
  } while (0)
#define KGE_DISPATCH_VEC(M, vec, CALL)          \
  do {                                          \
    if ((vec) == 4) { CALL(M, 4); }             \
    else if ((vec) == 2) { CALL(M, 2); }        \
    else { CALL(M, 1); }                        \
  } while (0)

}  // namespace kge
