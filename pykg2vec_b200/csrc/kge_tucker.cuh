// kge_tucker.cuh — kernels of TuckER's trunk (pykg2vec/models/projection.py:310-336), launched from kge_proj.cu.
//   tucker_gather_rows_kernel   relU[u, :] = rel[ids[u], :]: the A operand of the relation-level GEMMs
//   (the tiled GEMM of kge_proj.cuh)  M[u] = sum_k relU[u, k] W[k]: ONE core matrix per DISTINCT relation
//   tucker_trunk_fwd_kernel     gather + normalise + noise0 + contraction with M[slot] under the dropout1 mask +
//                               normalise + noise2, one CTA per query
//   tucker_trunk_bwd_kernel     its backward: the dense entity gradient and dM[slot] (atomics)
//   tucker_scatter_rows_kernel  grel[ids[u], :] += drelU[u, :]
//   tucker_mask1_kernel         the counter-mode dropout1 mask as a [Q, d1, d1] tensor (tests)
//
// Why per distinct relation: the reference builds W_mat = rel[r] @ W.view(d2, d1*d1) for every SAMPLE ([B, d1, d1],
// :321-323) and drops it out elementwise (:324).  The sum over k depends on the relation only and the mask acts
// after it, so x_pre[b, j] = sum_i ehat[b, i] m1[b, i, j] M[r_b][i, j] needs one M per distinct relation and no
// per-sample matrix; in counter mode the mask is regenerated from (seed, offset, element index) in forward and
// backward, so nothing of size B * d1 * d1 is read or written.
//
// Canonical arithmetic (DESIGN.md §3, TuckER):
//   M[u][c]   ONE sequential fma chain over k = 0 .. d2-1 from 0 (rule 8: the tiled GEMM's order, independent of
//             U and of the tiling)
//   sumsq     RSUM: 8 partials, element j -> partial (j >> 2) & 7 in increasing j by fma, butterfly 4, 2, 1
//   ehat[i]   = fmul(fdiv(ent[e][i], fmaxf(sqrt(sumsq), 1e-12)), noise0[i])       (F.normalize, then the dropout)
//   x_pre[j]  ONE sequential chain over i = 0 .. d1-1 from 0 of ffma(ehat[i], fmul(m1[i][j], M[i][j]), acc);
//             without a mask ffma(ehat[i], M[i][j], acc) (== a mask of ones, bit for bit)
//   x[j]      = fmul(fdiv(x_pre[j], fmaxf(sqrt(sumsq(x_pre)), 1e-12)), noise2[j])
//   m1        explicit: noise1[q][i][j].  counter: keep iff word 0 of Philox-4x32-10 with key (seed lo, seed hi)
//             and counter (lo, hi of offset + (q*d1 + i)*d1 + j, TUCKER_PHILOX_TAG, 0) is >= thresh(p); kept
//             elements are scaled by 1/(1-p) (tucker_mask_params)
// x is bit-exact against tests/oracle_tucker; the backward's sums over queries are float atomics in no fixed order.
#pragma once
#include "kge_proj.cuh"

namespace kge {

constexpr int TUCKER_THREADS = 256;
constexpr int TUCKER_MAX_D = 256;                  // widest d1 / d2: one thread per feature of a row
constexpr uint32_t TUCKER_PHILOX_TAG = 0x7475636bu;  // counter word 2: keeps these draws apart from ATen's streams
enum { TUCKER_MASK_NONE = 0, TUCKER_MASK_EXPLICIT = 1, TUCKER_MASK_COUNTER = 2 };

struct TuckerMask {
  int mode;
  const float* noise1;      // explicit: [Q, d1, d1]
  uint64_t seed, offset;    // counter
  uint32_t thresh;          // counter: keep iff draw >= thresh
  float scale;              // counter: value of a kept element
};

// thresh = ceil(p * 2^32) clamped to 2^32 - 1, scale = 1 / (float)(1 - p)  (p >= 1: everything dropped, as
// nn.Dropout(1.0) returns zeros)
inline void tucker_mask_params(float p, uint32_t* thresh, float* scale) {
  if (p >= 1.0f) { *thresh = 0xffffffffu; *scale = 0.f; return; }
  const double t = ceil((double)p * 4294967296.0);
  *thresh = t >= 4294967295.0 ? 0xffffffffu : (uint32_t)t;
  *scale = 1.0f / (float)(1.0 - (double)p);
}

// word 0 of Philox-4x32-10 (Salmon et al., SC'11) for key `seed` and counter (ctr lo, ctr hi, TAG, 0)
KGE_DEV uint32_t tucker_philox(uint64_t seed, uint64_t ctr) {
  uint32_t c0 = (uint32_t)ctr, c1 = (uint32_t)(ctr >> 32), c2 = TUCKER_PHILOX_TAG, c3 = 0u;
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  for (int r = 0; r < 10; ++r) {
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t n0 = (uint32_t)(p1 >> 32) ^ c1 ^ k0, n2 = (uint32_t)(p0 >> 32) ^ c3 ^ k1;
    c1 = (uint32_t)p1; c3 = (uint32_t)p0; c0 = n0; c2 = n2;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return c0;
}

// m1 of flat element idx = (q*d1 + i)*d1 + j (modes EXPLICIT and COUNTER)
KGE_DEV float tucker_mask_at(const TuckerMask& m, long long idx) {
  if (m.mode == TUCKER_MASK_EXPLICIT) return __ldg(m.noise1 + idx);
  return tucker_philox(m.seed, m.offset + (uint64_t)idx) >= m.thresh ? m.scale : 0.f;
}

// *out = sum_j a[j] * b[j] over shared-memory rows in the RSUM order, by threads 0..7 of the CTA (every thread
// calls it; barriers before and after are the caller's)
KGE_DEV void tucker_rsum(const float* a, const float* b, int n, float* out) {
  const int tid = threadIdx.x;
  if (tid < 8) {
    float acc = 0.f;
    for (int c = tid; 4 * c < n; c += 8)
      for (int e = 0; e < 4 && 4 * c + e < n; ++e) acc = ffma(a[4 * c + e], b[4 * c + e], acc);
    acc = group_sum(acc);
    if (tid == 0) *out = acc;
  }
}

__global__ void __launch_bounds__(256)
tucker_gather_rows_kernel(const float* __restrict__ rel, const int64_t* __restrict__ ids, long long U, int d2,
                          float* __restrict__ relU) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= U * d2) return;
  const long long u = i / d2;
  relU[i] = __ldg(rel + __ldg(ids + u) * d2 + (i - u * d2));
}

__global__ void __launch_bounds__(256)
tucker_scatter_rows_kernel(const float* __restrict__ drelU, const int64_t* __restrict__ ids, long long U, int d2,
                           float* __restrict__ grel) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i >= U * d2) return;
  const long long u = i / d2;
  atomicAdd(grel + __ldg(ids + u) * d2 + (i - u * d2), __ldg(drelU + i));
}

__global__ void __launch_bounds__(256)
tucker_mask1_kernel(TuckerMask m, long long n, float* __restrict__ out) {
  const long long i = (long long)blockIdx.x * 256 + threadIdx.x;
  if (i < n) out[i] = tucker_mask_at(m, i);
}

struct TuckerTrunk {
  const float* ent;         // [N, d1]
  const float* M;           // [U, d1*d1] core matrices
  const int64_t* e;         // [Q] entity ids
  const int64_t* slot;      // [Q] row of M of each query
  int d1;
  const float* noise0;      // [Q, d1] or NULL
  const float* noise2;      // [Q, d1] or NULL
  TuckerMask mask;
  float* x;                 // fwd out [Q, d1]
  float* xpre;              // fwd out (may be NULL) / bwd in: x before the second normalisation [Q, d1]
  float* nrm;               // fwd out (may be NULL) / bwd in: its L2 norm [Q]
  const float* gx;          // bwd in: d loss / d x [Q, d1]
  float* gent;              // bwd: dense [N, d1] gradient, accumulated (may be NULL)
  float* dM;                // bwd: [U, d1*d1], accumulated (may be NULL)
};

// one CTA per query, thread j owns feature j (d1 <= TUCKER_MAX_D = blockDim)
__global__ void __launch_bounds__(TUCKER_THREADS) tucker_trunk_fwd_kernel(const TuckerTrunk a) {
  __shared__ float es[TUCKER_MAX_D];
  __shared__ float xs[TUCKER_MAX_D];
  __shared__ float red[2];
  const int tid = threadIdx.x, d1 = a.d1;
  const long long q = blockIdx.x;
  const bool on = tid < d1;
  if (on) es[tid] = __ldg(a.ent + __ldg(a.e + q) * d1 + tid);
  __syncthreads();
  tucker_rsum(es, es, d1, &red[0]);
  __syncthreads();
  if (on) {
    float v = __fdiv_rn(es[tid], fmaxf(__fsqrt_rn(red[0]), 1e-12f));
    if (a.noise0) v = fmul(v, __ldg(a.noise0 + q * d1 + tid));
    es[tid] = v;   // threads 0..7 finished reading es before the barrier above
  }
  __syncthreads();
  if (on) {
    const float* Mq = a.M + __ldg(a.slot + q) * ((long long)d1 * d1) + tid;
    float acc = 0.f;
    if (a.mask.mode == TUCKER_MASK_NONE) {
      for (int i = 0; i < d1; ++i) acc = ffma(es[i], __ldg(Mq + (long long)i * d1), acc);
    } else {
      const long long base = q * d1 * (long long)d1 + tid;
      for (int i = 0; i < d1; ++i)
        acc = ffma(es[i], fmul(tucker_mask_at(a.mask, base + (long long)i * d1), __ldg(Mq + (long long)i * d1)), acc);
    }
    xs[tid] = acc;
    if (a.xpre) a.xpre[q * d1 + tid] = acc;
  }
  __syncthreads();
  tucker_rsum(xs, xs, d1, &red[1]);
  __syncthreads();
  const float n2 = __fsqrt_rn(red[1]);
  if (on) {
    float v = __fdiv_rn(xs[tid], fmaxf(n2, 1e-12f));
    if (a.noise2) v = fmul(v, __ldg(a.noise2 + q * d1 + tid));
    a.x[q * d1 + tid] = v;
  }
  if (a.nrm && tid == 0) a.nrm[q] = n2;
}

// y = v / max(n, eps) with n = ||v||:  dv = (dy - yhat (dy . yhat)) / n  while n > eps, else dy / eps
KGE_DEV float tucker_norm_bwd(float dy, float yhat, float dot, float n) {
  const float den = fmaxf(n, 1e-12f);
  return n > 1e-12f ? __fdiv_rn(fsub(dy, fmul(yhat, dot)), den) : __fdiv_rn(dy, den);
}

// one CTA per query.  Warp w owns the rows i = w, w+8, ... of the query's masked core matrix: its lanes walk the
// row (coalesced), accumulate dM[slot][i][j] += ehat[i] m1 g[j] and reduce d ehat[i] = sum_j m1 M[i][j] g[j]
__global__ void __launch_bounds__(TUCKER_THREADS) tucker_trunk_bwd_kernel(const TuckerTrunk a) {
  __shared__ float en[TUCKER_MAX_D];   // normalised entity row
  __shared__ float es[TUCKER_MAX_D];   // ehat = en * noise0
  __shared__ float g[TUCKER_MAX_D];    // d loss / d x_pre
  __shared__ float t0[TUCKER_MAX_D];
  __shared__ float t1[TUCKER_MAX_D];
  __shared__ float red[3];
  const int tid = threadIdx.x, d1 = a.d1, lane = tid & 31, warp = tid >> 5;
  const long long q = blockIdx.x;
  const bool on = tid < d1;
  const int64_t eid = __ldg(a.e + q);
  const float n2 = __ldg(a.nrm + q);
  if (on) {
    t0[tid] = __ldg(a.ent + eid * d1 + tid);
    const float gn = __ldg(a.gx + q * d1 + tid);
    g[tid] = a.noise2 ? fmul(gn, __ldg(a.noise2 + q * d1 + tid)) : gn;
    t1[tid] = __fdiv_rn(__ldg(a.xpre + q * d1 + tid), fmaxf(n2, 1e-12f));
  }
  __syncthreads();
  tucker_rsum(t0, t0, d1, &red[0]);
  tucker_rsum(g, t1, d1, &red[1]);
  __syncthreads();
  const float n1 = __fsqrt_rn(red[0]);
  if (on) {
    const float v = __fdiv_rn(t0[tid], fmaxf(n1, 1e-12f));
    en[tid] = v;
    es[tid] = a.noise0 ? fmul(v, __ldg(a.noise0 + q * d1 + tid)) : v;
    g[tid] = tucker_norm_bwd(g[tid], t1[tid], red[1], n2);
  }
  __syncthreads();
  const long long dd = (long long)d1 * d1;
  const float* Mq = a.M + __ldg(a.slot + q) * dd;
  float* dMq = a.dM ? a.dM + __ldg(a.slot + q) * dd : nullptr;
  for (int i = warp; i < d1; i += TUCKER_THREADS / 32) {
    const float ei = es[i];
    float acc = 0.f;
    for (int j = lane; j < d1; j += 32) {
      const long long o = (long long)i * d1 + j;
      const float gj = g[j];
      float w = __ldg(Mq + o), eg = ei;
      if (a.mask.mode != TUCKER_MASK_NONE) {
        const float m = tucker_mask_at(a.mask, q * dd + o);
        w = fmul(m, w);
        eg = fmul(ei, m);
      }
      acc = ffma(w, gj, acc);
      const float dm = fmul(eg, gj);
      if (dMq && dm != 0.f) atomicAdd(dMq + o, dm);
    }
#pragma unroll
    for (int off = 16; off; off >>= 1) acc = fadd(acc, __shfl_xor_sync(0xffffffffu, acc, off));
    if (lane == 0) t0[i] = acc;   // d ehat[i]; t0's earlier content was last read before the barrier above
  }
  __syncthreads();
  if (!a.gent) return;   // uniform over the CTA
  if (on && a.noise0) t0[tid] = fmul(t0[tid], __ldg(a.noise0 + q * d1 + tid));
  __syncthreads();
  tucker_rsum(t0, en, d1, &red[2]);
  __syncthreads();
  if (on) {
    const float d = tucker_norm_bwd(t0[tid], en[tid], red[2], n1);
    if (d != 0.f) atomicAdd(a.gent + eid * d1 + tid, d);
  }
}

// ---- launch plans of the relation-level GEMMs on proj_gemm_kernel (shared with tests/emu) -------------------
// M[U, d1*d1] = relU[U, d2] . W[d2, d1*d1]
inline ProjLaunch tucker_plan_cores(const float* relU, const float* W, long long U, int d1, int d2, float* M) {
  ProjLaunch L{};
  L.tile = PROJ_TILE_64x64;
  ProjGemm& g = L.g;
  const long long dd = (long long)d1 * d1;
  g.A = relU; g.sAm = d2; g.sAk = 1; g.Ap = nullptr;
  g.B = W; g.sBn = 1; g.sBk = dd;
  g.M = (int)U; g.N = (int)dd; g.K = d2; g.klen = (int)proj_tiles(d2, PBK) * PBK;
  g.avec = proj_vec_ok(relU, d2, 1); g.bvec = 0;
  g.C = M; g.ldc = dd; g.bias = nullptr; g.act = ACT_NONE;
  L.gx = proj_tiles(dd, PBN); L.gy = proj_tiles(U, PBM); L.gz = 1;
  return L;
}

// dW[d2, d1*d1] += relU^T[d2, U] . dM[U, d1*d1]   (one slice: every element receives exactly one atomic add)
inline ProjLaunch tucker_plan_grad_W(const float* relU, const float* dM, long long U, int d1, int d2, float* gW) {
  ProjLaunch L{};
  L.tile = PROJ_TILE_64x64;
  ProjGemm& g = L.g;
  const long long dd = (long long)d1 * d1;
  g.A = relU; g.sAm = 1; g.sAk = d2; g.Ap = nullptr;
  g.B = dM; g.sBn = 1; g.sBk = dd;
  g.M = d2; g.N = (int)dd; g.K = (int)U; g.klen = (int)proj_tiles(U, PBK) * PBK;
  g.avec = 0; g.bvec = 0;
  g.C = gW; g.ldc = dd;
  L.gx = proj_tiles(dd, PBN); L.gy = proj_tiles(d2, PBM); L.gz = 1;
  return L;
}

// drelU[U, d2] += dM[U, d1*d1] . W^T[d1*d1, d2]: contraction over d1*d1, split over `target_ctas` CTAs
inline ProjLaunch tucker_plan_grad_rel(const float* dM, const float* W, long long U, int d1, int d2, float* drelU,
                                       int target_ctas) {
  ProjLaunch L{};
  L.tile = PROJ_TILE_64x64;
  ProjGemm& g = L.g;
  const long long dd = (long long)d1 * d1;
  g.A = dM; g.sAm = dd; g.sAk = 1; g.Ap = nullptr;
  g.B = W; g.sBn = dd; g.sBk = 1;
  g.M = (int)U; g.N = d2; g.K = (int)dd;
  const long long tiles = (long long)proj_tiles(U, PBM) * proj_tiles(d2, PBN), chunks = proj_tiles(dd, PBK);
  long long splits = (target_ctas + tiles - 1) / tiles;
  if (splits > chunks) splits = chunks;
  if (splits < 1) splits = 1;
  const long long per = (chunks + splits - 1) / splits;
  g.klen = (int)(per * PBK);
  g.avec = proj_vec_ok(dM, dd, 1); g.bvec = proj_vec_ok(W, dd, 1);
  g.C = drelU; g.ldc = d2;
  L.gx = proj_tiles(d2, PBN); L.gy = proj_tiles(U, PBM); L.gz = (unsigned)((chunks + per - 1) / per);
  return L;
}

// workspace of kge_tucker_cores / kge_tucker_cores_bwd: relU and drelU, [U, d2] each
inline long long tucker_workspace_floats(long long U, int d2) { return 2 * (U > 0 ? U : 1) * (long long)d2; }

}  // namespace kge
