// kge_grads.cuh — per-model backward of the score functions, evaluated by an 8-lane
// group; replaces autograd through the reference's ATen chains (loss.backward(),
// pykg2vec/utils/trainer.py:298).  Intermediates are recomputed (nothing is saved
// by the forward), row gradients are accumulated with red.global.add (v4 when the
// row is 16-byte aligned) into dense gradient tables (nn.Embedding dense-grad
// semantics, pykg2vec/models/Domain.py:8-17).
//
// The backward differentiates forward() (TAIL grouping).  It is a floating-point
// path checked against the fp64 autograd oracle with a tolerance; it does not
// use the canonical-order intrinsics except where it recomputes forward values.
#pragma once
#include "kge_models.cuh"

namespace kge {

struct GradRows {
  float* h[8];
  float* t[8];
  float* r[8];
};

template <int MODEL>
KGE_DEV void resolve_grad_rows(GradRows& G, const ModelParams& P, float* const* gt, int64_t h,
                               int64_t r, int64_t t) {
  const size_t d = (size_t)P.d, dr = (size_t)P.dr;
#pragma unroll
  for (int c = 0; c < 8; ++c) G.h[c] = G.t[c] = G.r[c] = nullptr;
  auto at = [&](int k, size_t off) -> float* { return gt[k] ? gt[k] + off : nullptr; };
  if (MODEL == KGE_SLM || MODEL == KGE_NTN || MODEL == KGE_SME || MODEL == KGE_SME_BL || MODEL == KGE_CONVKB) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * dr);
    // dense parameters: whole gradient tables (not per-row)
#pragma unroll
    for (int k = 2; k < 8; ++k) G.r[k] = gt[k];
  } else if (MODEL == KGE_KG2E) {
    G.h[0] = at(0, h * d); G.h[1] = at(1, h * d); G.t[0] = at(0, t * d); G.t[1] = at(1, t * d);
    G.r[0] = at(2, r * d); G.r[1] = at(3, r * d);
  } else if (MODEL == KGE_QUATE || MODEL == KGE_OCTONIONE) {
    constexpr int C = (MODEL == KGE_QUATE) ? 4 : 8;
#pragma unroll
    for (int c = 0; c < C; ++c) { G.h[c] = at(c, h * d); G.t[c] = at(c, t * d); G.r[c] = at(C + c, r * d); }
  } else if (MODEL == KGE_ANALOGY) {
    const size_t d2 = d / 2;
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * d);
    G.h[1] = at(2, h * d2); G.h[2] = at(3, h * d2); G.t[1] = at(2, t * d2); G.t[2] = at(3, t * d2);
    G.r[1] = at(4, r * d2); G.r[2] = at(5, r * d2);
  } else if (MODEL == KGE_TRANSE || MODEL == KGE_DISTMULT || MODEL == KGE_TRANSM) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * d);
  } else if (MODEL == KGE_CP) {
    G.h[0] = at(0, h * d); G.t[0] = at(2, t * d); G.r[0] = at(1, r * d);
  } else if (MODEL == KGE_TRANSH) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * d); G.r[1] = at(2, r * d);
  } else if (MODEL == KGE_TRANSD) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * d);
    G.h[1] = at(2, h * d); G.t[1] = at(2, t * d); G.r[1] = at(3, r * d);
  } else if (MODEL == KGE_TRANSR) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * dr); G.r[1] = at(2, r * d * dr);
  } else if (MODEL == KGE_ROTATE) {
    G.h[0] = at(0, h * d); G.h[1] = at(1, h * d); G.t[0] = at(0, t * d); G.t[1] = at(1, t * d);
    G.r[0] = at(2, r * d);
  } else if (MODEL == KGE_COMPLEX) {
    G.h[0] = at(0, h * d); G.h[1] = at(1, h * d); G.t[0] = at(0, t * d); G.t[1] = at(1, t * d);
    G.r[0] = at(2, r * d); G.r[1] = at(3, r * d);
  } else if (MODEL == KGE_HOLE) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * d);
  } else if (MODEL == KGE_RESCAL) {
    G.h[0] = at(0, h * d); G.t[0] = at(0, t * d); G.r[0] = at(1, r * d * d);
  } else if (MODEL == KGE_SIMPLE || MODEL == KGE_SIMPLE_IGNR) {
    G.h[0] = at(0, h * d); G.h[1] = at(1, h * d); G.t[0] = at(1, t * d); G.t[1] = at(0, t * d);
    G.r[0] = at(2, r * d); G.r[1] = at(3, r * d);
  }
}

template <int VEC>
KGE_DEV void red_row_chunk(float* row, int c, int d, float4 g) {
  if (row) red_chunk<VEC>(row, c, d, g);
}

KGE_DEV float sgnf(float x) { return (x > 0.f) ? 1.f : ((x < 0.f) ? -1.f : 0.f); }

// Backward through  s = || h^ + r^ - t^ ||_p  with  v^ = v * inv_norm(v)   (F.normalize).
// fh/fr/ft(c): chunk c of the (already projected) operands.  gs = dL/ds.
struct DistCtx {
  float ih, ir, it;     // inverse norms
  float ch, cr, ct;     // coef * <v^, u>  per operand (projection term of normalize backward)
  float coef;           // gs (L1) or gs / s (L2)
  int l1;
};

template <class FH, class FR, class FT>
KGE_DEV DistCtx dist_prepare(FH fh, FR fr, FT ft, int nch, int lane, int l1, float gs) {
  DistCtx X;
  float sh = 0.f, sr = 0.f, st = 0.f;
  for (int c = lane; c < nch; c += 8) {
    const float4 a = fh(c), b = fr(c), cc = ft(c);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sh = ffma(f4_get(a, e), f4_get(a, e), sh);
      sr = ffma(f4_get(b, e), f4_get(b, e), sr);
      st = ffma(f4_get(cc, e), f4_get(cc, e), st);
    }
  }
  sh = group_sum(sh); sr = group_sum(sr); st = group_sum(st);
  X.ih = inv_norm_from_sumsq(sh); X.ir = inv_norm_from_sumsq(sr); X.it = inv_norm_from_sumsq(st);
  // norm below eps: F.normalize divides by the constant eps (clamp_min has zero gradient there)
  const bool clamp_h = __fsqrt_rn(sh) < 1e-12f, clamp_r = __fsqrt_rn(sr) < 1e-12f,
             clamp_t = __fsqrt_rn(st) < 1e-12f;
  X.l1 = l1;
  float S = 0.f, ah = 0.f, ar = 0.f, at = 0.f;
  for (int c = lane; c < nch; c += 8) {
    const float4 a = fh(c), b = fr(c), cc = ft(c);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float hn = f4_get(a, e) * X.ih, rn = f4_get(b, e) * X.ir, tn = f4_get(cc, e) * X.it;
      const float x = (hn + rn) - tn;
      const float u = l1 ? sgnf(x) : x;
      S += x * x; ah += hn * u; ar += rn * u; at += tn * u;
    }
  }
  S = group_sum(S); ah = group_sum(ah); ar = group_sum(ar); at = group_sum(at);
  const float s = sqrtf(S);
  X.coef = l1 ? gs : ((s > 0.f) ? gs / s : 0.f);
  X.ch = clamp_h ? 0.f : X.coef * ah;
  X.cr = clamp_r ? 0.f : X.coef * ar;
  X.ct = clamp_t ? 0.f : X.coef * at;
  return X;
}

// gradient w.r.t. one element of each operand given its raw values
KGE_DEV void dist_elem(const DistCtx& X, float hv, float rv, float tv, float& dh, float& dr, float& dt) {
  const float hn = hv * X.ih, rn = rv * X.ir, tn = tv * X.it;
  const float x = (hn + rn) - tn;
  const float dx = X.coef * (X.l1 ? sgnf(x) : x);
  dh = (dx - hn * X.ch) * X.ih;
  dr = (dx - rn * X.cr) * X.ir;
  dt = -(dx - tn * X.ct) * X.it;
}

// TransE / TransM backward with the three rows held in registers (CH chunks per lane, as load_trans_chunks
// fills them): norms, projections and the scatter from registers.
template <int CH, int VEC>
KGE_DEV void grad_trans_regs(const float4 (&A)[CH], const float4 (&B)[CH], const float4 (&C)[CH], const GradRows& G,
                             int d, int nch, int lane, int l1, float gs) {
  DistCtx X;
  float sh = 0.f, sr = 0.f, st = 0.f;
#pragma unroll
  for (int k = 0; k < CH; ++k)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      sh = ffma(f4_get(A[k], e), f4_get(A[k], e), sh);
      sr = ffma(f4_get(B[k], e), f4_get(B[k], e), sr);
      st = ffma(f4_get(C[k], e), f4_get(C[k], e), st);
    }
  sh = group_sum(sh); sr = group_sum(sr); st = group_sum(st);
  X.ih = inv_norm_from_sumsq(sh); X.ir = inv_norm_from_sumsq(sr); X.it = inv_norm_from_sumsq(st);
  const bool clamp_h = __fsqrt_rn(sh) < 1e-12f, clamp_r = __fsqrt_rn(sr) < 1e-12f, clamp_t = __fsqrt_rn(st) < 1e-12f;
  X.l1 = l1;
  float S = 0.f, ah = 0.f, ar = 0.f, at = 0.f;
#pragma unroll
  for (int k = 0; k < CH; ++k)
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float hn = f4_get(A[k], e) * X.ih, rn = f4_get(B[k], e) * X.ir, tn = f4_get(C[k], e) * X.it;
      const float x = (hn + rn) - tn;
      const float u = l1 ? sgnf(x) : x;
      S += x * x; ah += hn * u; ar += rn * u; at += tn * u;
    }
  S = group_sum(S); ah = group_sum(ah); ar = group_sum(ar); at = group_sum(at);
  const float s = sqrtf(S);
  X.coef = l1 ? gs : ((s > 0.f) ? gs / s : 0.f);
  X.ch = clamp_h ? 0.f : X.coef * ah;
  X.cr = clamp_r ? 0.f : X.coef * ar;
  X.ct = clamp_t ? 0.f : X.coef * at;
#pragma unroll
  for (int k = 0; k < CH; ++k) {
    const int c = lane + 8 * k;
    if (c < nch) {
      float4 dh, dr, dt;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        dist_elem(X, f4_get(A[k], e), f4_get(B[k], e), f4_get(C[k], e), f4_at(dh, e), f4_at(dr, e), f4_at(dt, e));
      red_row_chunk<VEC>(G.h[0], c, d, dh);
      red_row_chunk<VEC>(G.r[0], c, d, dr);
      red_row_chunk<VEC>(G.t[0], c, d, dt);
    }
  }
}

// ... with one trip to memory for the operands
template <int CH, int VEC>
KGE_DEV void grad_trans_cached(const TripleRows& R, const GradRows& G, int d, int nch, int lane, int l1,
                               float gs) {
  float4 A[CH], B[CH], C[CH];
  load_trans_chunks<CH>([&](int c) { return ld_chunk<VEC>(R.h[0], c, d); },
                        [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); },
                        [&](int c) { return ld_chunk<VEC>(R.t[0], c, d); }, nch, lane, A, B, C);
  grad_trans_regs<CH, VEC>(A, B, C, G, d, nch, lane, l1, gs);
}

// Accumulate gs * d score / d rows into G.  All 8 lanes call; `scratch` per group
// (group_scratch_floats_bwd floats, TransR only).
template <int MODEL, int VEC, int CHSEL = -1>
KGE_DEV void grad_group(const TripleRows& R, const GradRows& G, const ModelParams& P, int lane,
                        float gs, float* scratch) {
  const int d = P.d;
  const int nch = (d + 3) >> 2;
  if (MODEL == KGE_TRANSE || MODEL == KGE_TRANSM) {
    if (MODEL == KGE_TRANSM) gs *= __ldg(R.r[1]);
    if (CHSEL > 0) { grad_trans_cached<(CHSEL > 0 ? CHSEL : 1), VEC>(R, G, d, nch, lane, P.l1, gs); return; }
    if (CHSEL < 0) {
      if (nch <= 16) { grad_trans_cached<2, VEC>(R, G, d, nch, lane, P.l1, gs); return; }
      if (nch <= 32) { grad_trans_cached<4, VEC>(R, G, d, nch, lane, P.l1, gs); return; }
      if (nch <= 64) { grad_trans_cached<8, VEC>(R, G, d, nch, lane, P.l1, gs); return; }
    }
    auto fh = [&](int c) { return ld_chunk<VEC>(R.h[0], c, d); };
    auto fr = [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); };
    auto ft = [&](int c) { return ld_chunk<VEC>(R.t[0], c, d); };
    const DistCtx X = dist_prepare(fh, fr, ft, nch, lane, P.l1, gs);
    for (int c = lane; c < nch; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c);
      float4 dh, dr, dt;
#pragma unroll
      for (int e = 0; e < 4; ++e)
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), f4_at(dh, e), f4_at(dr, e), f4_at(dt, e));
      red_row_chunk<VEC>(G.h[0], c, d, dh);
      red_row_chunk<VEC>(G.r[0], c, d, dr);
      red_row_chunk<VEC>(G.t[0], c, d, dt);
    }
  } else if (MODEL == KGE_TRANSH) {
    float sw = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 w = ld_chunk<VEC>(R.r[1], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) sw = ffma(f4_get(w, e), f4_get(w, e), sw);
    }
    sw = group_sum(sw);
    const float iw = inv_norm_from_sumsq(sw);
    const bool clamp_w = __fsqrt_rn(sw) < 1e-12f;
    float ah = 0.f, at = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 w = ld_chunk<VEC>(R.r[1], c, d), a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float wn = fmul(f4_get(w, e), iw);
        ah = ffma(f4_get(a, e), wn, ah);
        at = ffma(f4_get(b, e), wn, at);
      }
    }
    ah = group_sum(ah); at = group_sum(at);
    auto wn4 = [&](int c) {
      const float4 w = ld_chunk<VEC>(R.r[1], c, d);
      return make_float4(fmul(w.x, iw), fmul(w.y, iw), fmul(w.z, iw), fmul(w.w, iw));
    };
    auto proj = [&](const float* row, float a, int c) {
      const float4 w = wn4(c), x = ld_chunk<VEC>(row, c, d);
      float4 o;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(o, e) = ffma(-a, f4_get(w, e), f4_get(x, e));
      return o;
    };
    auto fh = [&](int c) { return proj(R.h[0], ah, c); };
    auto fr = [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); };
    auto ft = [&](int c) { return proj(R.t[0], at, c); };
    const DistCtx X = dist_prepare(fh, fr, ft, nch, lane, P.l1, gs);
    // bh = <w~, dh_perp>, bt = <w~, dt_perp>
    float bh = 0.f, bt = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c), w = wn4(c);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float dh, dr, dt;
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), dh, dr, dt);
        bh += f4_get(w, e) * dh; bt += f4_get(w, e) * dt;
      }
    }
    bh = group_sum(bh); bt = group_sum(bt);
    // cw = <w~, dw~>,  dw~_k = -h_k bh - ah dh_perp_k - t_k bt - at dt_perp_k
    float cw = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c), w = wn4(c);
      const float4 hv = ld_chunk<VEC>(R.h[0], c, d), tv = ld_chunk<VEC>(R.t[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float dh, dr, dt;
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), dh, dr, dt);
        const float dwn = -f4_get(hv, e) * bh - ah * dh - f4_get(tv, e) * bt - at * dt;
        cw += f4_get(w, e) * dwn;
      }
    }
    cw = group_sum(cw);
    if (clamp_w) cw = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c), w = wn4(c);
      const float4 hv = ld_chunk<VEC>(R.h[0], c, d), tv = ld_chunk<VEC>(R.t[0], c, d);
      float4 gh, gr, gtt, gw;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float dh, dr, dt;
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), dh, dr, dt);
        const float dwn = -f4_get(hv, e) * bh - ah * dh - f4_get(tv, e) * bt - at * dt;
        f4_at(gh, e) = dh - f4_get(w, e) * bh;
        f4_at(gtt, e) = dt - f4_get(w, e) * bt;
        f4_at(gr, e) = dr;
        f4_at(gw, e) = (dwn - f4_get(w, e) * cw) * iw;
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
      red_row_chunk<VEC>(G.r[1], c, d, gw);
    }
  } else if (MODEL == KGE_TRANSD) {
    const float ah = group_dot<VEC>(R.h[0], R.h[1], d, nch, lane);
    const float at = group_dot<VEC>(R.t[0], R.t[1], d, nch, lane);
    auto proj = [&](const float* row, float a, int c) {
      const float4 rm = ld_chunk<VEC>(R.r[1], c, d), x = ld_chunk<VEC>(row, c, d);
      float4 o;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(o, e) = ffma(a, f4_get(rm, e), f4_get(x, e));
      return o;
    };
    auto fh = [&](int c) { return proj(R.h[0], ah, c); };
    auto fr = [&](int c) { return ld_chunk<VEC>(R.r[0], c, d); };
    auto ft = [&](int c) { return proj(R.t[0], at, c); };
    const DistCtx X = dist_prepare(fh, fr, ft, nch, lane, P.l1, gs);
    float bh = 0.f, bt = 0.f;  // <r_m, dh'>, <r_m, dt'>
    for (int c = lane; c < nch; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c), rm = ld_chunk<VEC>(R.r[1], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float dh, dr, dt;
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), dh, dr, dt);
        bh += f4_get(rm, e) * dh; bt += f4_get(rm, e) * dt;
      }
    }
    bh = group_sum(bh); bt = group_sum(bt);
    for (int c = lane; c < nch; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c);
      const float4 hv = ld_chunk<VEC>(R.h[0], c, d), tv = ld_chunk<VEC>(R.t[0], c, d),
                   hm = ld_chunk<VEC>(R.h[1], c, d), tm = ld_chunk<VEC>(R.t[1], c, d);
      float4 gh, gr, gtt, ghm, gtm, grm;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float dh, dr, dt;
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), dh, dr, dt);
        f4_at(gh, e) = dh + f4_get(hm, e) * bh;
        f4_at(gtt, e) = dt + f4_get(tm, e) * bt;
        f4_at(ghm, e) = f4_get(hv, e) * bh;
        f4_at(gtm, e) = f4_get(tv, e) * bt;
        f4_at(gr, e) = dr;
        f4_at(grm, e) = ah * dh + at * dt;
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
      red_row_chunk<VEC>(G.h[1], c, d, ghm);
      red_row_chunk<VEC>(G.t[1], c, d, gtm);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
      red_row_chunk<VEC>(G.r[1], c, d, grm);
    }
  } else if (MODEL == KGE_ROTATE) {
    const float g2 = 2.f * gs;
    for (int c = lane; c < nch; c += 8) {
      const float4 hr = ld_chunk<VEC>(R.h[0], c, d), hi = ld_chunk<VEC>(R.h[1], c, d),
                   rr = ld_chunk<VEC>(R.r[0], c, d), tr = ld_chunk<VEC>(R.t[0], c, d),
                   ti = ld_chunk<VEC>(R.t[1], c, d);
      float4 ghr, ghi, gtr, gti, grr;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float im, re;
        sincos_canon(fmul(f4_get(rr, e), P.phase), im, re);
        const float sr = f4_get(hr, e) * re - f4_get(hi, e) * im - f4_get(tr, e);
        const float si = f4_get(hr, e) * im + f4_get(hi, e) * re - f4_get(ti, e);
        const float dsr = g2 * sr, dsi = g2 * si;
        f4_at(ghr, e) = dsr * re + dsi * im;
        f4_at(ghi, e) = -dsr * im + dsi * re;
        f4_at(gtr, e) = -dsr;
        f4_at(gti, e) = -dsi;
        const float dre = dsr * f4_get(hr, e) + dsi * f4_get(hi, e);
        const float dim = -dsr * f4_get(hi, e) + dsi * f4_get(hr, e);
        f4_at(grr, e) = (-dre * im + dim * re) * P.phase;
      }
      red_row_chunk<VEC>(G.h[0], c, d, ghr);
      red_row_chunk<VEC>(G.h[1], c, d, ghi);
      red_row_chunk<VEC>(G.t[0], c, d, gtr);
      red_row_chunk<VEC>(G.t[1], c, d, gti);
      red_row_chunk<VEC>(G.r[0], c, d, grr);
    }
  } else if (MODEL == KGE_DISTMULT || MODEL == KGE_CP) {
    const float ng = -gs;
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.r[0], c, d), cc = ld_chunk<VEC>(R.t[0], c, d);
      float4 gh, gr, gtt;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        f4_at(gh, e) = ng * f4_get(b, e) * f4_get(cc, e);
        f4_at(gr, e) = ng * f4_get(a, e) * f4_get(cc, e);
        f4_at(gtt, e) = ng * f4_get(a, e) * f4_get(b, e);
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
    }
  } else if (MODEL == KGE_CONVKB) {
    // s = <a_h,h> + <a_r,r> + <a_t,t> + c0:  d row = gs * a ;  d a += gs * row ;  d c0 += gs
    const float* A = P.tab[2];
    float* gA = G.r[2];
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.r[0], c, d), cc = ld_chunk<VEC>(R.t[0], c, d);
      const float4 wa = ld_chunk<VEC>(A, c, d), wb = ld_chunk<VEC>(A + d, c, d), wc = ld_chunk<VEC>(A + 2 * (size_t)d, c, d);
      float4 gh, gr, gtt, ga, gb, gc;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        f4_at(gh, e) = gs * f4_get(wa, e); f4_at(gr, e) = gs * f4_get(wb, e); f4_at(gtt, e) = gs * f4_get(wc, e);
        f4_at(ga, e) = gs * f4_get(a, e); f4_at(gb, e) = gs * f4_get(b, e); f4_at(gc, e) = gs * f4_get(cc, e);
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
      if (gA) { red_chunk<VEC>(gA, c, d, ga); red_chunk<VEC>(gA + d, c, d, gb); red_chunk<VEC>(gA + 2 * (size_t)d, c, d, gc); }
    }
    if (lane == 0 && G.r[3]) atomicAdd(G.r[3], gs);
  } else if (MODEL == KGE_COMPLEX) {
    const float ng = -gs;
    for (int c = lane; c < nch; c += 8) {
      const float4 hr = ld_chunk<VEC>(R.h[0], c, d), hi = ld_chunk<VEC>(R.h[1], c, d),
                   rr = ld_chunk<VEC>(R.r[0], c, d), ri = ld_chunk<VEC>(R.r[1], c, d),
                   tr = ld_chunk<VEC>(R.t[0], c, d), ti = ld_chunk<VEC>(R.t[1], c, d);
      float4 ghr, ghi, grr, gri, gtr, gti;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float a = f4_get(hr, e), b = f4_get(hi, e), p = f4_get(rr, e), q = f4_get(ri, e),
                    x = f4_get(tr, e), y = f4_get(ti, e);
        f4_at(ghr, e) = ng * (x * p + y * q);
        f4_at(ghi, e) = ng * (y * p - x * q);
        f4_at(gtr, e) = ng * (a * p - b * q);
        f4_at(gti, e) = ng * (b * p + a * q);
        f4_at(grr, e) = ng * (a * x + b * y);
        f4_at(gri, e) = ng * (a * y - b * x);
      }
      red_row_chunk<VEC>(G.h[0], c, d, ghr);
      red_row_chunk<VEC>(G.h[1], c, d, ghi);
      red_row_chunk<VEC>(G.r[0], c, d, grr);
      red_row_chunk<VEC>(G.r[1], c, d, gri);
      red_row_chunk<VEC>(G.t[0], c, d, gtr);
      red_row_chunk<VEC>(G.t[1], c, d, gti);
    }
  } else if (MODEL == KGE_SLM || MODEL == KGE_NTN) {
    // s = -sum_k r^_k tanh(pre_k).  scratch: [6 dm forward pieces] dpre, dhn, dtn  (dm each)
    const int K = P.dr, nchk = (K + 3) >> 2, dm = dense_dm(d, K);
    DenseCtx X;
    slm_ntn_fill<MODEL, VEC>(R, P, lane, scratch, X);
    float *dpre = scratch + 6 * dm, *dhn = scratch + 7 * dm, *dtn = scratch + 8 * dm;
    float* gmr1 = G.r[2]; float* gmr2 = G.r[3];
    const float ng = -gs;
    float rdot = 0.f;
    for (int c = lane; c < nchk; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = 4 * c + e;
        const float a = X.act[k], rk = X.rn[k];
        dpre[k] = (k < K) ? ng * rk * (1.f - a * a) : 0.f;
        rdot += rk * (ng * a);
      }
    }
    for (int c = lane; c < nch; c += 8) { *reinterpret_cast<float4*>(dhn + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f); *reinterpret_cast<float4*>(dtn + 4 * c) = make_float4(0.f, 0.f, 0.f, 0.f); }
    rdot = group_sum(rdot);
    if (X.clamp_r) rdot = 0.f;
    group_sync();
    // relation row: d r = (d r^ - r^ <r^, d r^>) * ir,  d r^_k = ng * act_k
    for (int c = lane; c < nchk; c += 8) {
      float4 gr;
#pragma unroll
      for (int e = 0; e < 4; ++e) { const int k = 4 * c + e; f4_at(gr, e) = (ng * X.act[k] - X.rn[k] * rdot) * X.ir; }
      red_row_chunk<VEC>(G.r[0], c, K, gr);
      if (MODEL == KGE_NTN && G.r[4]) red_chunk<VEC>(G.r[4], c, K, *reinterpret_cast<const float4*>(dpre + 4 * c));
    }
    // linear layers: d hn_i += sum_k mr1[i,k] dpre_k ; d mr1[i,k] += hn_i dpre_k (same for t / mr2)
    const float* mr1 = P.tab[2];
    const float* mr2 = P.tab[3];
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * c + e;
        if (i >= d) continue;
        float ah = 0.f, at = 0.f;
        const float hi = X.hn[i], ti = X.tn[i];
        for (int kc = 0; kc < nchk; ++kc) {
          const float4 m1 = ld_chunk<VEC>(mr1 + (size_t)i * K, kc, K), m2 = ld_chunk<VEC>(mr2 + (size_t)i * K, kc, K);
          const float4 dp = *reinterpret_cast<const float4*>(dpre + 4 * kc);
          float4 g1, g2;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            ah += f4_get(m1, q) * f4_get(dp, q); at += f4_get(m2, q) * f4_get(dp, q);
            f4_at(g1, q) = hi * f4_get(dp, q); f4_at(g2, q) = ti * f4_get(dp, q);
          }
          if (gmr1) red_chunk<VEC>(gmr1 + (size_t)i * K, kc, K, g1);
          if (gmr2) red_chunk<VEC>(gmr2 + (size_t)i * K, kc, K, g2);
        }
        dhn[i] += ah; dtn[i] += at;
      }
    }
    if (MODEL == KGE_NTN) {
      // bilinear tensor: pre_k += h^T W_k t^ :  d hn_i += dpre_k sum_j W[i,j] tn_j ; d tn_j += dpre_k sum_i hn_i W[i,j]
      //                                         d W_k[i,j] += dpre_k hn_i tn_j
      group_sync();
      for (int k = 0; k < K; ++k) {
        const float dk = dpre[k];
        const float* W = P.tab[5] + (size_t)k * d * d;
        float* gW = G.r[5] ? G.r[5] + (size_t)k * d * d : nullptr;
        for (int c = lane; c < nch; c += 8) {       // lane owns columns j = 4c..4c+3
          const float4 tt = *reinterpret_cast<const float4*>(X.tn + 4 * c);
          float4 accj = make_float4(0.f, 0.f, 0.f, 0.f);
          for (int i = 0; i < d; ++i) {
            const float hi = X.hn[i];
            const float4 w = ld_chunk<VEC>(W + (size_t)i * d, c, d);
            float4 gw;
            float rowdot = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
              f4_at(accj, q) += hi * f4_get(w, q);
              rowdot += f4_get(w, q) * f4_get(tt, q);
              f4_at(gw, q) = dk * hi * f4_get(tt, q);
            }
            if (gW) red_chunk<VEC>(gW + (size_t)i * d, c, d, gw);
            atomicAdd(dhn + i, dk * rowdot);   // shared-memory accumulate across the lanes' column chunks
          }
#pragma unroll
          for (int q = 0; q < 4; ++q) if (4 * c + q < d) dtn[4 * c + q] += dk * f4_get(accj, q);
        }
        group_sync();
      }
    }
    group_sync();
    float hdot = 0.f, tdot = 0.f;
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) { const int i = 4 * c + e; if (i < d) { hdot += X.hn[i] * dhn[i]; tdot += X.tn[i] * dtn[i]; } }
    }
    hdot = group_sum(hdot); tdot = group_sum(tdot);
    if (X.clamp_h) hdot = 0.f;
    if (X.clamp_t) tdot = 0.f;
    for (int c = lane; c < nch; c += 8) {
      float4 gh, gtt;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * c + e;
        f4_at(gh, e) = (i < d) ? (dhn[i] - X.hn[i] * hdot) * X.ih : 0.f;
        f4_at(gtt, e) = (i < d) ? (dtn[i] - X.tn[i] * tdot) * X.it : 0.f;
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
    }
    group_sync();
  } else if (MODEL == KGE_SME || MODEL == KGE_SME_BL) {
    // scratch: [9 dm forward pieces] dhn, drn, dtn
    const int dm = nch * 4;
    DenseCtx X;
    sme_fill<MODEL, VEC>(R, P, lane, scratch, X);
    float *dhn = scratch + 9 * dm, *drn = scratch + 10 * dm, *dtn = scratch + 11 * dm;
    for (int c = lane; c < nch; c += 8) {
      const float4 z = make_float4(0.f, 0.f, 0.f, 0.f);
      *reinterpret_cast<float4*>(dhn + 4 * c) = z; *reinterpret_cast<float4*>(drn + 4 * c) = z; *reinterpret_cast<float4*>(dtn + 4 * c) = z;
    }
    group_sync();
    const float ng = (MODEL == KGE_SME) ? -gs : gs;
    const float *mu1 = P.tab[2], *mu2 = P.tab[3], *mv1 = P.tab[5], *mv2 = P.tab[6];
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int k = 4 * c + e;
        if (k >= d) continue;
        const float dgu = ng * X.gv[k], dgv = ng * X.gu[k];
        float du1, du2, dv1, dv2;
        if (MODEL == KGE_SME) { du1 = du2 = dgu; dv1 = dv2 = dgv; }
        else { du1 = dgu * X.u2[k]; du2 = dgu * X.u1[k]; dv1 = dgv * X.v2[k]; dv2 = dgv * X.v1[k]; }
        if (G.r[4]) atomicAdd(G.r[4] + k, dgu);
        if (G.r[7]) atomicAdd(G.r[7] + k, dgv);
        const size_t ro = (size_t)k * d;
        for (int i = 0; i < d; ++i) {
          const float hi = X.hn[i], ri = X.rn[i], ti = X.tn[i];
          atomicAdd(dhn + i, __ldg(mu1 + ro + i) * du1);
          atomicAdd(drn + i, __ldg(mu2 + ro + i) * du2 + __ldg(mv2 + ro + i) * dv2);
          atomicAdd(dtn + i, __ldg(mv1 + ro + i) * dv1);
          if (G.r[2]) atomicAdd(G.r[2] + ro + i, du1 * hi);
          if (G.r[3]) atomicAdd(G.r[3] + ro + i, du2 * ri);
          if (G.r[5]) atomicAdd(G.r[5] + ro + i, dv1 * ti);
          if (G.r[6]) atomicAdd(G.r[6] + ro + i, dv2 * ri);
        }
      }
    }
    group_sync();
    float hdot = 0.f, tdot = 0.f, rdot = 0.f;
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * c + e;
        if (i < d) { hdot += X.hn[i] * dhn[i]; tdot += X.tn[i] * dtn[i]; rdot += X.rn[i] * drn[i]; }
      }
    }
    hdot = group_sum(hdot); tdot = group_sum(tdot); rdot = group_sum(rdot);
    if (X.clamp_h) hdot = 0.f;
    if (X.clamp_t) tdot = 0.f;
    if (X.clamp_r) rdot = 0.f;
    for (int c = lane; c < nch; c += 8) {
      float4 gh, gtt, gr;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int i = 4 * c + e;
        f4_at(gh, e) = (i < d) ? (dhn[i] - X.hn[i] * hdot) * X.ih : 0.f;
        f4_at(gtt, e) = (i < d) ? (dtn[i] - X.tn[i] * tdot) * X.it : 0.f;
        f4_at(gr, e) = (i < d) ? (drn[i] - X.rn[i] * rdot) * X.ir : 0.f;
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
    }
    group_sync();
  } else if (MODEL == KGE_KG2E) {
    // rows k: 0 h_mu, 1 h_sigma, 2 r_mu, 3 r_sigma, 4 t_mu, 5 t_sigma; y^ = y / ||y||
    const float* rows6[6] = {R.h[0], R.h[1], R.r[0], R.r[1], R.t[0], R.t[1]};
    float* grows6[6] = {G.h[0], G.h[1], G.r[0], G.r[1], G.t[0], G.t[1]};
    float inv[6], dot[6];
#pragma unroll
    for (int k = 0; k < 6; ++k) {
      float s = 0.f;
      for (int c = lane; c < nch; c += 8) {
        const float4 x = ld_chunk<VEC>(rows6[k], c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) s = ffma(f4_get(x, e), f4_get(x, e), s);
      }
      inv[k] = __frcp_rn(__fsqrt_rn(group_sum(s)));
      dot[k] = 0.f;
    }
    // d score / d normalised operands at element j
    auto elem = [&](int j, float (&y)[6], float (&dy)[6]) {
#pragma unroll
      for (int k = 0; k < 6; ++k) y[k] = __ldg(rows6[k] + j) * inv[k];
      const float cs = y[1] + y[3], cm = y[0] + y[2], st = y[5], x = y[4] - cm;
      const float ist = 1.f / st, ics = 1.f / cs;
      dy[0] = -2.f * x * ist; dy[2] = dy[0]; dy[4] = 2.f * x * ist;
      dy[1] = ist - ics; dy[3] = dy[1];
      dy[5] = (-(cs + x * x) * ist + 1.f) * ist;
    };
    for (int c = lane; c < nch; c += 8)
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        if (j >= d) continue;
        float y[6], dy[6];
        elem(j, y, dy);
#pragma unroll
        for (int k = 0; k < 6; ++k) dot[k] += y[k] * dy[k];
      }
#pragma unroll
    for (int k = 0; k < 6; ++k) dot[k] = group_sum(dot[k]);
    for (int c = lane; c < nch; c += 8)
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        if (j >= d) continue;
        float y[6], dy[6];
        elem(j, y, dy);
#pragma unroll
        for (int k = 0; k < 6; ++k)
          if (grows6[k]) atomicAdd(grows6[k] + j, gs * (dy[k] - y[k] * dot[k]) * inv[k]);
      }
  } else if (MODEL == KGE_QUATE || MODEL == KGE_OCTONIONE) {
    // score = -sum_j <h (x) r^, t>:  d t = -gs * o;  (d h, d r^) through the (bi)linear product;
    // d r through the per-dimension unit-modulus normalisation.  Scalar atomics (rows are strided).
    constexpr int C = (MODEL == KGE_QUATE) ? 4 : 8;
    const float ng = -gs;
    for (int c = lane; c < nch; c += 8) {
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        if (j >= d) continue;
        float hc[C], rc[C], tc[C], o[C], dh[C], drn[C];
        float inv;
#pragma unroll
        for (int k = 0; k < C; ++k) { hc[k] = __ldg(R.h[k] + j); rc[k] = __ldg(R.r[k] + j); tc[k] = __ldg(R.t[k] + j); }
        hyper_product<C>(hc, rc, o, &inv);   // rc now holds r^
        // dO = ng * t
        float dO[C];
#pragma unroll
        for (int k = 0; k < C; ++k) dO[k] = ng * tc[k];
        auto qmult_bwd = [](const float* A, const float* B, const float* g, float* dA, float* dB, float sA, float sB) {
          // out = qmult(A, B); accumulate sA * dA, sB * dB (pointers may be null)
          if (dA) {
            dA[0] += sA * ( g[0] * B[0] + g[1] * B[1] + g[2] * B[2] + g[3] * B[3]);
            dA[1] += sA * (-g[0] * B[1] + g[1] * B[0] - g[2] * B[3] + g[3] * B[2]);
            dA[2] += sA * (-g[0] * B[2] + g[1] * B[3] + g[2] * B[0] - g[3] * B[1]);
            dA[3] += sA * (-g[0] * B[3] - g[1] * B[2] + g[2] * B[1] + g[3] * B[0]);
          }
          if (dB) {
            dB[0] += sB * ( g[0] * A[0] + g[1] * A[1] + g[2] * A[2] + g[3] * A[3]);
            dB[1] += sB * (-g[0] * A[1] + g[1] * A[0] + g[2] * A[3] - g[3] * A[2]);
            dB[2] += sB * (-g[0] * A[2] - g[1] * A[3] + g[2] * A[0] + g[3] * A[1]);
            dB[3] += sB * (-g[0] * A[3] + g[1] * A[2] - g[2] * A[1] + g[3] * A[0]);
          }
        };
#pragma unroll
        for (int k = 0; k < C; ++k) { dh[k] = 0.f; drn[k] = 0.f; }
        if (C == 4) {
          qmult_bwd(hc, rc, dO, dh, drn, 1.f, 1.f);
        } else {
          const float dstar[4] = {rc[4], -rc[5], -rc[6], -rc[7]}, cstar[4] = {rc[0], -rc[1], -rc[2], -rc[3]};
          float gds[4] = {0.f, 0.f, 0.f, 0.f}, gcs[4] = {0.f, 0.f, 0.f, 0.f};
          // o[0..3] = qmult(a, c) - qmult(d*, b);   o[4..7] = qmult(d, a) + qmult(b, c*)
          qmult_bwd(hc, rc, dO, dh, drn, 1.f, 1.f);                   // a, c
          qmult_bwd(dstar, hc + 4, dO, gds, dh + 4, -1.f, -1.f);      // d*, b  (minus sign)
          qmult_bwd(rc + 4, hc, dO + 4, drn + 4, dh, 1.f, 1.f);       // d, a
          qmult_bwd(hc + 4, cstar, dO + 4, dh + 4, gcs, 1.f, 1.f);    // b, c*
          drn[4] += gds[0]; drn[5] -= gds[1]; drn[6] -= gds[2]; drn[7] -= gds[3];
          drn[0] += gcs[0]; drn[1] -= gcs[1]; drn[2] -= gcs[2]; drn[3] -= gcs[3];
        }
        float dot = 0.f;
#pragma unroll
        for (int k = 0; k < C; ++k) dot += rc[k] * drn[k];
#pragma unroll
        for (int k = 0; k < C; ++k) {
          if (G.h[k]) atomicAdd(G.h[k] + j, dh[k]);
          if (G.t[k]) atomicAdd(G.t[k] + j, ng * o[k]);
          if (G.r[k]) atomicAdd(G.r[k] + j, (drn[k] - rc[k] * dot) * inv);
        }
      }
    }
  } else if (MODEL == KGE_ANALOGY) {
    const float ng = -gs;
    const int d2 = d / 2, nch2 = (d2 + 3) >> 2;
    for (int c = lane; c < nch2; c += 8) {
      const float4 hr = ld_chunk<VEC>(R.h[1], c, d2), hi = ld_chunk<VEC>(R.h[2], c, d2),
                   rr = ld_chunk<VEC>(R.r[1], c, d2), ri = ld_chunk<VEC>(R.r[2], c, d2),
                   tr = ld_chunk<VEC>(R.t[1], c, d2), ti = ld_chunk<VEC>(R.t[2], c, d2);
      float4 ghr, ghi, grr, gri, gtr, gti;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const float a = f4_get(hr, e), b = f4_get(hi, e), p = f4_get(rr, e), q = f4_get(ri, e),
                    x = f4_get(tr, e), y = f4_get(ti, e);
        f4_at(ghr, e) = ng * (x * p + y * q);
        f4_at(ghi, e) = ng * (y * p - x * q);
        f4_at(gtr, e) = ng * (a * p - b * q);
        f4_at(gti, e) = ng * (b * p + a * q);
        f4_at(grr, e) = ng * (a * x + b * y);
        f4_at(gri, e) = ng * (a * y - b * x);
      }
      red_row_chunk<VEC>(G.h[1], c, d2, ghr); red_row_chunk<VEC>(G.h[2], c, d2, ghi);
      red_row_chunk<VEC>(G.r[1], c, d2, grr); red_row_chunk<VEC>(G.r[2], c, d2, gri);
      red_row_chunk<VEC>(G.t[1], c, d2, gtr); red_row_chunk<VEC>(G.t[2], c, d2, gti);
    }
    for (int c = lane; c < nch; c += 8) {
      const float4 a = ld_chunk<VEC>(R.h[0], c, d), b = ld_chunk<VEC>(R.r[0], c, d), cc = ld_chunk<VEC>(R.t[0], c, d);
      float4 gh, gr, gtt;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        f4_at(gh, e) = ng * f4_get(b, e) * f4_get(cc, e);
        f4_at(gr, e) = ng * f4_get(a, e) * f4_get(cc, e);
        f4_at(gtt, e) = ng * f4_get(a, e) * f4_get(b, e);
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
    }
  } else if (MODEL == KGE_SIMPLE || MODEL == KGE_SIMPLE_IGNR) {
    const float half = (MODEL == KGE_SIMPLE) ? 0.5f : 1.0f;
    float acc = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 h1 = ld_chunk<VEC>(R.h[0], c, d), t2 = ld_chunk<VEC>(R.h[1], c, d),
                   t1 = ld_chunk<VEC>(R.t[0], c, d), h2 = ld_chunk<VEC>(R.t[1], c, d),
                   r1 = ld_chunk<VEC>(R.r[0], c, d), r2 = ld_chunk<VEC>(R.r[1], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e)
        acc += f4_get(h1, e) * f4_get(r1, e) * f4_get(t1, e) + half * f4_get(h2, e) * f4_get(r2, e) * f4_get(t2, e);
    }
    const float init = group_sum(acc);
    // -clamp(init, -20, 20): gradient passes only inside the clamp range (torch.clamp backward)
    const float ng = (init >= -20.f && init <= 20.f) ? -gs : 0.f;
    const float ngh = ng * half;
    for (int c = lane; c < nch; c += 8) {
      const float4 h1 = ld_chunk<VEC>(R.h[0], c, d), t2 = ld_chunk<VEC>(R.h[1], c, d),
                   t1 = ld_chunk<VEC>(R.t[0], c, d), h2 = ld_chunk<VEC>(R.t[1], c, d),
                   r1 = ld_chunk<VEC>(R.r[0], c, d), r2 = ld_chunk<VEC>(R.r[1], c, d);
      float4 gh1, gt2, gt1, gh2, gr1, gr2;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        f4_at(gh1, e) = ng * f4_get(r1, e) * f4_get(t1, e);
        f4_at(gr1, e) = ng * f4_get(h1, e) * f4_get(t1, e);
        f4_at(gt1, e) = ng * f4_get(h1, e) * f4_get(r1, e);
        f4_at(gh2, e) = ngh * f4_get(r2, e) * f4_get(t2, e);
        f4_at(gr2, e) = ngh * f4_get(h2, e) * f4_get(t2, e);
        f4_at(gt2, e) = ngh * f4_get(h2, e) * f4_get(r2, e);
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh1);
      red_row_chunk<VEC>(G.h[1], c, d, gt2);
      red_row_chunk<VEC>(G.t[0], c, d, gt1);
      red_row_chunk<VEC>(G.t[1], c, d, gh2);
      red_row_chunk<VEC>(G.r[0], c, d, gr1);
      red_row_chunk<VEC>(G.r[1], c, d, gr2);
    }
  } else if (MODEL == KGE_RESCAL) {
    // s = -h^T M t:  dh_j = -gs (M t)_j ; dt_k = -gs (h^T M)_k ; dM_jk = -gs h_j t_k
    const float* M = R.r[0];
    const float ng = -gs;
    for (int c = lane; c < nch; c += 8) {
      float4 v = make_float4(0.f, 0.f, 0.f, 0.f);   // (h^T M) chunk c
      const float4 tc = ld_chunk<VEC>(R.t[0], c, d);
      for (int j = 0; j < d; ++j) {
        const float hj = __ldg(R.h[0] + j);
        const float4 mrow = ld_chunk<VEC>(M + (size_t)j * d, c, d);
        float4 gm;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          f4_at(v, e) += hj * f4_get(mrow, e);
          f4_at(gm, e) = ng * hj * f4_get(tc, e);
        }
        if (G.r[0]) red_chunk<VEC>(G.r[0] + (size_t)j * d, c, d, gm);
      }
      float4 gt;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(gt, e) = ng * f4_get(v, e);
      red_row_chunk<VEC>(G.t[0], c, d, gt);
    }
    for (int c = lane; c < nch; c += 8) {           // (M t) rows j in chunk c
      float4 u = make_float4(0.f, 0.f, 0.f, 0.f);
      for (int kc = 0; kc < nch; ++kc) {
        const float4 tv = ld_chunk<VEC>(R.t[0], kc, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const int j = 4 * c + e;
          if (j < d) {
            const float4 mrow = ld_chunk<VEC>(M + (size_t)j * d, kc, d);
#pragma unroll
            for (int q = 0; q < 4; ++q) f4_at(u, e) += f4_get(mrow, q) * f4_get(tv, q);
          }
        }
      }
      float4 gh;
#pragma unroll
      for (int e = 0; e < 4; ++e) f4_at(gh, e) = ng * f4_get(u, e);
      red_row_chunk<VEC>(G.h[0], c, d, gh);
    }
  } else if (MODEL == KGE_HOLE) {
    // s = sum_k r^_k e_k, e = circconv(eh, et), score = -sigmoid(s).
    // scratch: rn, eh, et, deh, det, dr  [dp each]
    const int dp = nch * 4;
    float *rn = scratch, *eh = rn + dp, *et = eh + dp, *deh = et + dp, *det = deh + dp, *drn = det + dp;
    float sr = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 b = ld_chunk<VEC>(R.r[0], c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) sr = ffma(f4_get(b, e), f4_get(b, e), sr);
    }
    sr = group_sum(sr);
    const float ir = inv_norm_from_sumsq(sr);
    const bool clamp_r = __fsqrt_rn(sr) < 1e-12f;
    for (int c = lane; c < nch; c += 8) {
      const float4 b = ld_chunk<VEC>(R.r[0], c, d);
      *reinterpret_cast<float4*>(rn + 4 * c) = make_float4(b.x * ir, b.y * ir, b.z * ir, b.w * ir);
      *reinterpret_cast<float4*>(eh + 4 * c) = even_chunk(R.h[0], c, d);
      *reinterpret_cast<float4*>(et + 4 * c) = even_chunk(R.t[0], c, d);
    }
    group_sync();
    // deh[n] = sum_m et[m] rn[(m+n)%d]; det[m] = sum_n eh[n] rn[(m+n)%d]; drn[j] = sum_n eh[n] et[(j-n)%d]
    float s_part = 0.f;
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int a = 4 * c + e;
        float x = 0.f, y = 0.f, z = 0.f;
        if (a < d) {
          int idx = a, back = a;
          for (int b = 0; b < d; ++b) {
            x += et[b] * rn[idx];
            y += eh[b] * rn[idx];
            z += eh[b] * et[back];
            idx = (idx + 1 == d) ? 0 : idx + 1;
            back = (back == 0) ? d - 1 : back - 1;
          }
          s_part += rn[a] * z;
        }
        deh[a] = x; det[a] = y; drn[a] = z;
      }
    }
    const float sv = group_sum(s_part);
    const float sg = 1.f / (1.f + expf(-sv));
    const float gp = -gs * sg * (1.f - sg);
    group_sync();
    float rdot = 0.f;
    for (int c = lane; c < nch; c += 8) {
#pragma unroll
      for (int e = 0; e < 4; ++e) { const int j = 4 * c + e; if (j < d) rdot += rn[j] * drn[j]; }
    }
    rdot = group_sum(rdot);
    if (clamp_r) rdot = 0.f;
    for (int c = lane; c < nch; c += 8) {
      float4 gh, gt, gr;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        if (j < d) {
          const int jm = (j == 0) ? 0 : d - j;
          f4_at(gh, e) = gp * 0.5f * (deh[j] + deh[jm]);
          f4_at(gt, e) = gp * 0.5f * (det[j] + det[jm]);
          f4_at(gr, e) = gp * (drn[j] - rn[j] * rdot) * ir;
        } else { f4_at(gh, e) = 0.f; f4_at(gt, e) = 0.f; f4_at(gr, e) = 0.f; }
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.t[0], c, d, gt);
      red_row_chunk<VEC>(G.r[0], c, d, gr);
    }
    group_sync();
  } else if (MODEL == KGE_TRANSR) {
    // h^ = h*ih; h'_k = sum_j h^_j M_jk; h'^ = normalise(h'); r^ = normalise(r) (then normalised
    // again inside the distance); x = h'^ + r^^ - t'^.   scratch: hp, tp, dhp, dtp [drp each],
    // dhn, dtn [dp each]  (see group_scratch_floats_bwd).
    const int dr = P.dr, nchr = (dr + 3) >> 2, drp = nchr * 4, dp = nch * 4;
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
    sh = group_sum(sh); st = group_sum(st); sr = group_sum(sr);
    const float ih = inv_norm_from_sumsq(sh), it = inv_norm_from_sumsq(st), ir = inv_norm_from_sumsq(sr);
    const bool clamp_h0 = __fsqrt_rn(sh) < 1e-12f, clamp_t0 = __fsqrt_rn(st) < 1e-12f,
               clamp_r0 = __fsqrt_rn(sr) < 1e-12f;
    float* hp = scratch;
    float* tp = hp + drp;
    float* dhp = tp + drp;
    float* dtp = dhp + drp;
    float* dhn = dtp + drp;  // [dp] gradient w.r.t. normalised head
    float* dtn = dhn + dp;
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
    auto fh = [&](int c) { return *reinterpret_cast<const float4*>(hp + 4 * c); };
    auto fr = [&](int c) {
      const float4 b = ld_chunk<VEC>(R.r[0], c, dr);
      return make_float4(fmul(b.x, ir), fmul(b.y, ir), fmul(b.z, ir), fmul(b.w, ir));
    };
    auto ft = [&](int c) { return *reinterpret_cast<const float4*>(tp + 4 * c); };
    const DistCtx X = dist_prepare(fh, fr, ft, nchr, lane, P.l1, gs);
    float rdot = 0.f;  // <r^, dr^>
    for (int c = lane; c < nchr; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c);
      float4 dh, drn, dt;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), f4_at(dh, e), f4_at(drn, e), f4_at(dt, e));
        rdot += f4_get(b, e) * f4_get(drn, e);
      }
      *reinterpret_cast<float4*>(dhp + 4 * c) = dh;
      *reinterpret_cast<float4*>(dtp + 4 * c) = dt;
    }
    rdot = group_sum(rdot);
    if (clamp_r0) rdot = 0.f;
    for (int c = lane; c < nchr; c += 8) {
      const float4 a = fh(c), b = fr(c), cc = ft(c);
      float4 gr;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        float dh, drn, dt;
        dist_elem(X, f4_get(a, e), f4_get(b, e), f4_get(cc, e), dh, drn, dt);
        f4_at(gr, e) = (drn - f4_get(b, e) * rdot) * ir;
      }
      red_row_chunk<VEC>(G.r[0], c, dr, gr);
    }
    // dh^_j = sum_k M_jk dh'_k ; dM_jk = h^_j dh'_k + t^_j dt'_k
    float hdot = 0.f, tdot = 0.f;
    for (int j = 0; j < d; ++j) {
      const float hn = fmul(__ldg(R.h[0] + j), ih), tn = fmul(__ldg(R.t[0] + j), it);
      float ph = 0.f, pt = 0.f;
      for (int c = lane; c < nchr; c += 8) {
        const float4 mrow = ld_chunk<VEC>(R.r[1] + (size_t)j * dr, c, dr);
        const float4 dh = *reinterpret_cast<const float4*>(dhp + 4 * c);
        const float4 dt = *reinterpret_cast<const float4*>(dtp + 4 * c);
        float4 gm;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          ph += f4_get(mrow, e) * f4_get(dh, e);
          pt += f4_get(mrow, e) * f4_get(dt, e);
          f4_at(gm, e) = hn * f4_get(dh, e) + tn * f4_get(dt, e);
        }
        if (G.r[1]) red_chunk<VEC>(G.r[1] + (size_t)j * dr, c, dr, gm);
      }
      ph = group_sum(ph); pt = group_sum(pt);
      hdot += hn * ph; tdot += tn * pt;
      if (lane == 0) { dhn[j] = ph; dtn[j] = pt; }
    }
    if (clamp_h0) hdot = 0.f;
    if (clamp_t0) tdot = 0.f;
    group_sync();   // this group's lanes only: callers branch per group (train_hinge_kernel: active pairs)
    for (int c = lane; c < nch; c += 8) {
      const float4 hv = ld_chunk<VEC>(R.h[0], c, d), tv = ld_chunk<VEC>(R.t[0], c, d);
      float4 gh, gtt;
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int j = 4 * c + e;
        const float a = (j < d) ? dhn[j] : 0.f, b = (j < d) ? dtn[j] : 0.f;
        f4_at(gh, e) = (a - f4_get(hv, e) * ih * hdot) * ih;
        f4_at(gtt, e) = (b - f4_get(tv, e) * it * tdot) * it;
      }
      red_row_chunk<VEC>(G.h[0], c, d, gh);
      red_row_chunk<VEC>(G.t[0], c, d, gtt);
    }
    (void)dp;
  }
}

// shared-memory floats one 8-lane group needs in the backward kernels
inline size_t group_scratch_floats_bwd(const kge_model_t* m) {
  if (m->model == KGE_SLM || m->model == KGE_NTN) return 9 * (size_t)dense_dm(m->dim, m->rel_dim);
  if (m->model == KGE_SME || m->model == KGE_SME_BL) return 12 * (size_t)(((m->dim + 3) >> 2) * 4);
  if (m->model == KGE_HOLE) return 6 * (size_t)(((m->dim + 3) >> 2) * 4);
  if (m->model == KGE_RESCAL) return group_scratch_floats(m);
  if (m->model != KGE_TRANSR) return 0;
  const size_t drp = (size_t)(((m->rel_dim + 3) >> 2) * 4), dp = (size_t)(((m->dim + 3) >> 2) * 4);
  return 4 * drp + 2 * dp;
}

}  // namespace kge
