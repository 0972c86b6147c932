// kge_rank_tiled.cu — shared-memory tiled 1-vs-all sweep (the dominant kernel of evaluation).
//
// For a block of QBLK queries and a run of candidate rows, every (query, candidate) score is
// evaluated from on-chip operands and compared with the query's threshold (its target's
// score); only per-query counts leave the SM.  The arithmetic per pair is exactly the
// canonical order of DESIGN.md §3 — an 8-lane group owns a register tile of TQ x TC pairs,
// lane l accumulates the chunks l, l+8, ... of the embedding axis, and the cross-lane
// butterfly (4,2,1) is done as a reduce-scatter so that each lane finishes a different pair —
// hence bit-identical to kge_score_fwd / the gather sweep / the CPU oracle.
//
// Data movement: operand tiles are staged in shared memory by 2-D TMA tensor-map loads
// (cp.async.bulk.tensor.2d, completion on an mbarrier; UTMALDG.2D in SASS), double buffered;
// out-of-range rows / columns arrive zero-filled.  A tile is stored OCTET-MAJOR: one {32 columns
// x rows} box per octet of the embedding axis lands as [octet][row][32 floats], so a group's 8
// lanes read 128 contiguous bytes (conflict-free for every width) and every address in the
// compute loop is a per-lane base plus a compile-time immediate.  Query vectors are prepared
// once per call (prep_query_kernel, which also yields the thresholds) into a compact
// [Q][KQ][dp] buffer; candidates come straight from the model tables (or from a normalised /
// even-part / padded scratch copy; raw TransE rows are normalised in shared memory).  Two modes,
// chosen on the host from the shared-memory budget: whole rows (query block resident for the whole
// CTA) and slabs of DS <= 256 columns for wide models (d = 500, 1000), accumulators living across slabs.
//
// Bound: fp32 pipe (2-8 instructions per element pair), not HBM: a candidate row is read from
// L2 once per query BLOCK instead of once per query.
#include "kge_models.cuh"
#include "kge_rank.cuh"
#include "kge_rank_resolve.cuh"
#include "kge_rank_tc.cuh"
#include "kge_tma.cuh"

namespace kge {

constexpr int kTThreads = 256;
constexpr int kTGroups = kTThreads / 8;  // 32
constexpr int kGQ = 16;                  // query sub-blocks per CTA
constexpr int kGC = kTGroups / kGQ;      // 2 candidate group columns
constexpr int kNT = 4;                   // register tiles (candidate sub-blocks) per group
constexpr int kTC = 4;                   // candidates per register tile
constexpr int kCBLK = kGC * kNT * kTC;   // 32 candidates per tile

enum { OP_TRANS_T = 0, OP_TRANS_H = 1, OP_DOT1 = 2, OP_DOT2 = 3, OP_ROT = 4 };

template <int OP> struct OpTraits { static constexpr int KQ = 1, KC = 1, TQ = 4; };
template <> struct OpTraits<OP_DOT2> { static constexpr int KQ = 2, KC = 2, TQ = 4; };
template <> struct OpTraits<OP_ROT> { static constexpr int KQ = 2, KC = 2, TQ = 4; };

struct TiledParams {
  const float* qvec;      // [Q][KQ][dp]
  const float* cand[2];   // KC candidate arrays, row pitch cand_pitch floats
  int64_t cand_pitch;
  const float* cand_inv;  // TransE on the raw table: [nc] inverse row norms the staged rows are scaled by, or nullptr
  const float* thr;       // [Q]
  const float* qscale;    // [Q] (TransM theta[r]) or nullptr
  int64_t Q, nc;
  int dp, DS, nslabs;
  int tiles_per_cta, ntiles;
  int splits, units;      // work unit u = (run of tiles u % splits, query block u / splits); units = splits x blocks
  int32_t* counts;
  int col, l1;
  int fin;      // DOT ops: 0 -> -sum ; 1 -> -sigmoid(sum) (HoLE) ; 2 -> -clamp(sum, +-20) (SimplE)
  float margin;
};

// ---- per-element pair operations (canonical arithmetic) ---------------------------------------
// Two-term models (DOT2, ROT) accumulate chunk-wise — the chunk's 4 first terms, then its 4
// second terms (DESIGN.md §3 rule 6) — so the two operand halves are consumed one after the other
// and never have to be live in registers together.
template <int OP, bool L1>
KGE_DEV void pair_op(float& acc, const float4* q, const float4* c) {
  if (OP == OP_TRANS_T || OP == OP_TRANS_H) {
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float x = (OP == OP_TRANS_T) ? fsub(f4_get(q[0], e), f4_get(c[0], e))
                                         : fadd(f4_get(c[0], e), f4_get(q[0], e));
      if (L1) acc = fadd(acc, fabsf(x)); else acc = ffma(x, x, acc);
    }
  } else if (OP == OP_DOT1) {
#pragma unroll
    for (int e = 0; e < 4; ++e) acc = ffma(f4_get(q[0], e), f4_get(c[0], e), acc);
  } else if (OP == OP_DOT2) {
#pragma unroll
    for (int e = 0; e < 4; ++e) acc = ffma(f4_get(q[0], e), f4_get(c[0], e), acc);
#pragma unroll
    for (int e = 0; e < 4; ++e) acc = ffma(f4_get(q[1], e), f4_get(c[1], e), acc);
  } else {  // OP_ROT: |q - c|^2 over (re, im); q = h o r (tail sweep) or t o conj(r) (head sweep)
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float sr = fsub(f4_get(q[0], e), f4_get(c[0], e)); acc = ffma(sr, sr, acc); }
#pragma unroll
    for (int e = 0; e < 4; ++e) { const float si = fsub(f4_get(q[1], e), f4_get(c[1], e)); acc = ffma(si, si, acc); }
  }
}

template <int OP, bool L1>
KGE_DEV float finalize(float sum, float qscale, float margin, bool has_scale, int fin) {
  if (OP == OP_TRANS_T || OP == OP_TRANS_H) {
    if (L1 || !has_scale) return sum;                // L2 without a scale: threshold is in the sum domain
    return fmul(qscale, __fsqrt_rn(sum));
  }
  if (OP == OP_DOT1 || OP == OP_DOT2) {
    if (fin == 1) return -sigmoid_canon(sum);
    if (fin == 2) return -fminf(fmaxf(sum, -20.0f), 20.0f);
    return -sum;
  }
  return fsub(sum, margin);
}

// Butterfly 4,2,1 over the group's 8 lanes as a reduce-scatter: on return v[0 .. NV/8) hold
// complete sums of the pairs  orig = b4*NV/2 + b2*NV/4 + b1*NV/8 + i  (b* = lane bits 2,1,0).
template <int NV>
KGE_DEV void reduce_scatter(float (&v)[NV], int lane) {
  const unsigned m = 0xffffffffu;  // the whole warp is converged here; xor 4/2/1 stays inside the 8-lane group
  {
    const bool hi = lane & 4;
#pragma unroll
    for (int i = 0; i < NV / 2; ++i) {
      const float send = hi ? v[i] : v[i + NV / 2];
      const float keep = hi ? v[i + NV / 2] : v[i];
      v[i] = fadd(keep, __shfl_xor_sync(m, send, 4));
    }
  }
  {
    const bool hi = lane & 2;
#pragma unroll
    for (int i = 0; i < NV / 4; ++i) {
      const float send = hi ? v[i] : v[i + NV / 4];
      const float keep = hi ? v[i + NV / 4] : v[i];
      v[i] = fadd(keep, __shfl_xor_sync(m, send, 2));
    }
  }
  {
    const bool hi = lane & 1;
#pragma unroll
    for (int i = 0; i < NV / 8; ++i) {
      const float send = hi ? v[i] : v[i + NV / 8];
      const float keep = hi ? v[i + NV / 8] : v[i];
      v[i] = fadd(keep, __shfl_xor_sync(m, send, 1));
    }
  }
}

struct TiledMaps { CUtensorMap q, c0, c1; };

template <int OP, bool L1>
__device__ __forceinline__ void sweep_tiled_body(const TiledParams& P, const TiledMaps& TM, int unit) {
  constexpr int KQ = OpTraits<OP>::KQ, KC = OpTraits<OP>::KC, TQ = OpTraits<OP>::TQ;
  constexpr int QBLK = kGQ * TQ;
  constexpr int NV = TQ * kTC;
  constexpr int kWarps = kTThreads / 32;
  extern __shared__ __align__(128) unsigned char smem_raw[];
  // layout: [2 mbarriers][2 stage-release counters][thr QBLK][qs QBLK][cnt QBLK] | q stages | c stages
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw);
  unsigned* s_done = reinterpret_cast<unsigned*>(smem_raw + 16);
  float* s_thr = reinterpret_cast<float*>(smem_raw + 32);
  float* s_qs = s_thr + QBLK;
  int* s_cnt = reinterpret_cast<int*>(s_qs + QBLK);
  const int hdr = ((32 + 3 * QBLK * 4) + 127) / 128 * 128;
  const int DS = P.DS;
  const int qstages = P.nslabs > 1 ? 2 : 1;
  // thread mapping: the 4 groups of a warp share the candidate column group `gc` and cover 4
  // adjacent query sub-blocks (`warp` comes through a shuffle so that it is known to be uniform)
  const int tid = threadIdx.x, lane = tid & 7, lane32 = tid & 31;
  const int warp = __shfl_sync(0xffffffffu, tid >> 5, 0);
  const int g = (tid >> 3) & 3;
  const int gc = warp % kGC, gq = (warp / kGC) * 4 + g;
  const int64_t q0 = (int64_t)(unit / P.splits) * QBLK;
  const int qrows = (int)min((int64_t)QBLK, P.Q - q0);
  const int t0 = (unit % P.splits) * P.tiles_per_cta;
  const int ntile_local = min(P.tiles_per_cta, P.ntiles - t0);
  if (ntile_local <= 0) return;
  const int T = ntile_local * P.nslabs;
  const bool sum_domain = (OP == OP_TRANS_T || OP == OP_TRANS_H) && !L1 && P.qscale == nullptr;

  if (tid < QBLK) {
    // rows beyond Q get a threshold no score is below, so they never count
    float th = tid < qrows ? __ldg(P.thr + q0 + tid) : -INFINITY;
    if (sum_domain) th = sqrt_domain_threshold(th);
    s_thr[tid] = th;
    s_qs[tid] = (tid < qrows && P.qscale) ? __ldg(P.qscale + q0 + tid) : 1.f;
    s_cnt[tid] = 0;
  }
  if (tid == 0) {
    mbar_init(&bars[0], 1);
    mbar_init(&bars[1], 1);
    s_done[0] = 0u;
    s_done[1] = 0u;
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  // producer: ONE WARP issues the TMA loads of iteration `it` into stage it&1.  A tile is stored
  // OCTET-MAJOR — [octet of 32 columns][row][32 floats] — by one {32 x rows} box per octet and
  // operand (lanes 0..noct-1 issue one octet each), so that every shared-memory address of the
  // compute loop is  per-lane base + compile-time immediate  whatever the embedding width is.
  // Out-of-range rows / columns arrive as zeros.
  constexpr uint32_t kQOct = (uint32_t)(QBLK * KQ) * 128u;     // bytes of one query octet  [QBLK*KQ][32]
  constexpr uint32_t kCOct = (uint32_t)(KC * kCBLK) * 128u;    // bytes of one candidate octet [KC][CBLK][32]
  const uint32_t q_stage_bytes = (uint32_t)(QBLK * KQ) * (uint32_t)DS * 4u;
  const uint32_t c_stage_bytes = (uint32_t)(KC * kCBLK) * (uint32_t)DS * 4u;
  unsigned char* const qbase = smem_raw + hdr;
  unsigned char* const cbase = qbase + (size_t)qstages * q_stage_bytes;
  auto issue = [&](int it) {   // called by all 32 lanes of one warp
    const int stage = it & 1;
    const int tile = t0 + it / P.nslabs, slab = it % P.nslabs;
    const bool load_q = (P.nslabs > 1) || (it == 0);
    const int noct = (min(DS, P.dp - slab * DS) + 31) >> 5;
    if (lane32 == 0)
      mbar_arrive_expect_tx(&bars[stage], (uint32_t)noct * (kCOct + (load_q ? kQOct : 0u)));
    __syncwarp();
    if (lane32 < noct) {
      unsigned char* cdst = cbase + (size_t)stage * c_stage_bytes + (size_t)lane32 * kCOct;
      const int col = slab * DS + 32 * lane32;
      tma_load_2d(smem_u32(cdst), &TM.c0, col, tile * kCBLK, &bars[stage]);
      if (KC == 2) tma_load_2d(smem_u32(cdst + (size_t)kCBLK * 128u), &TM.c1, col, tile * kCBLK, &bars[stage]);
      if (load_q)
        tma_load_2d(smem_u32(qbase + (size_t)(P.nslabs > 1 ? stage : 0) * q_stage_bytes + (size_t)lane32 * kQOct),
                    &TM.q, col, (int)(q0 * KQ), &bars[stage]);
    }
  };

  // which pair(s) this lane finishes after the reduce-scatter, and its (fixed) query row
  const int b4 = (lane >> 2) & 1, b2 = (lane >> 1) & 1, b1 = lane & 1;
  const int orig0 = b4 * (NV / 2) + b2 * (NV / 4) + b1 * (NV / 8);
  const int my_iq = orig0 / kTC;                 // same for all of the lane's results
  const int qrow = gq * TQ + my_iq;
  const float th = s_thr[qrow], qsc = s_qs[qrow];
  const bool has_scale = P.qscale != nullptr;
  int cnt = 0;

  float acc[kNT][NV];
  if (warp == 0) {
    issue(0);
    if (T > 1) issue(1);
  }
  int tile = t0, slab = 0;
  for (int it = 0; it < T; ++it) {
    const int stage = it & 1;
    if (slab == 0) {
#pragma unroll
      for (int nt = 0; nt < kNT; ++nt)
#pragma unroll
        for (int i = 0; i < NV; ++i) acc[nt][i] = 0.f;
    }
    mbar_wait(&bars[stage], (uint32_t)((it >> 1) & 1));
    if constexpr (OP == OP_TRANS_T || OP == OP_TRANS_H) {
      if (P.cand_inv) {
        // raw TransE rows: normalise the staged candidate tile once, with prep_cand_kernel's fmul(x, inv) (same
        // bits as the scratch copy; columns past the row are zeros either way, rows past nc are left alone)
        float* ct = reinterpret_cast<float*>(cbase + (size_t)stage * c_stage_bytes);
        const int64_t r0 = (int64_t)tile * kCBLK;
        const int nel = ((min(DS, P.dp - slab * DS) + 31) >> 5) * kCBLK * 32;   // [octet][row][32 floats]
        for (int i = tid; i < nel; i += kTThreads) {
          const int64_t row = r0 + ((i >> 5) % kCBLK);
          if (row < P.nc) ct[i] = fmul(ct[i], __ldg(P.cand_inv + row));
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // before the stage's next TMA refill
        __syncthreads();
      }
    }
    const int nch = min(DS, P.dp - slab * DS) >> 2;
    // lane's chunk c = 8*octet + lane of row r sits at  octet*OctBytes + r*128 + lane*16
    const unsigned char* qs = qbase + (size_t)(P.nslabs > 1 ? stage : 0) * q_stage_bytes + (gq * TQ * KQ) * 128 + lane * 16;
    const unsigned char* cs = cbase + (size_t)stage * c_stage_bytes + (gc * kTC) * 128 + lane * 16;
#pragma unroll 1
    for (int c = lane; c < nch; c += 8, qs += kQOct, cs += kCOct) {
      if constexpr (OP == OP_DOT2 || OP == OP_ROT) {
        // two-term ops: all first-term operands, then all second-term operands — every accumulator
        // still sees its chunk's 4 first terms before its 4 second terms, and only one half of
        // the operands is live at a time (fits 2 CTAs per SM)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          float4 qk[TQ];
#pragma unroll
          for (int i = 0; i < TQ; ++i) qk[i] = *reinterpret_cast<const float4*>(qs + (i * KQ + k) * 128);
#pragma unroll
          for (int nt = 0; nt < kNT; ++nt) {
            float4 ck[kTC];
#pragma unroll
            for (int j = 0; j < kTC; ++j)
              ck[j] = *reinterpret_cast<const float4*>(cs + (k * kCBLK + kGC * kTC * nt + j) * 128);
#pragma unroll
            for (int i = 0; i < TQ; ++i)
#pragma unroll
              for (int j = 0; j < kTC; ++j) {
                float& a = acc[nt][i * kTC + j];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  if (OP == OP_DOT2) a = ffma(f4_get(qk[i], e), f4_get(ck[j], e), a);
                  else { const float x = fsub(f4_get(qk[i], e), f4_get(ck[j], e)); a = ffma(x, x, a); }
                }
              }
          }
        }
      } else {
        float4 q4[TQ][KQ];
#pragma unroll
        for (int i = 0; i < TQ; ++i)
#pragma unroll
          for (int k = 0; k < KQ; ++k)
            q4[i][k] = *reinterpret_cast<const float4*>(qs + (i * KQ + k) * 128);
#pragma unroll
        for (int nt = 0; nt < kNT; ++nt) {
          float4 c4[kTC][KC];
#pragma unroll
          for (int j = 0; j < kTC; ++j)
#pragma unroll
            for (int k = 0; k < KC; ++k)
              c4[j][k] = *reinterpret_cast<const float4*>(cs + (k * kCBLK + kGC * kTC * nt + j) * 128);
#pragma unroll
          for (int i = 0; i < TQ; ++i)
#pragma unroll
            for (int j = 0; j < kTC; ++j) pair_op<OP, L1>(acc[nt][i * kTC + j], q4[i], c4[j]);
        }
      }
    }
    // Stage recycling without a CTA barrier: every warp bumps the stage's release counter when it
    // has read its last operand of this iteration; the warp that arrives last (count % kWarps ==
    // kWarps-1) refills the stage with iteration it+2.  No warp ever waits for another warp —
    // only for data.
    __syncwarp();
    {
      unsigned prev = 0u;
      if (lane32 == 0) {
        __threadfence_block();
        prev = atomicAdd(&s_done[stage], 1u);
        __threadfence_block();
      }
      prev = __shfl_sync(0xffffffffu, prev, 0);
      if ((prev % kWarps) == kWarps - 1 && it + 2 < T) issue(it + 2);
    }
    if (slab == P.nslabs - 1) {
      // candidates of this tile that exist (the last tile may be ragged; missing rows are zeros)
      const int nvalid = (int)min((int64_t)kCBLK, P.nc - (int64_t)tile * kCBLK);
#pragma unroll
      for (int nt = 0; nt < kNT; ++nt) {
        reduce_scatter<NV>(acc[nt], lane);
#pragma unroll
        for (int i = 0; i < NV / 8; ++i) {
          const int jc = (orig0 + i) % kTC;
          const int local = (gc + kGC * nt) * kTC + jc;
          const float s = finalize<OP, L1>(acc[nt][i], qsc, P.margin, has_scale, P.fin);
          cnt += (local < nvalid && s < th) ? 1 : 0;
        }
      }
    }
    if (++slab == P.nslabs) { slab = 0; ++tile; }
  }
  if (cnt) atomicAdd(&s_cnt[qrow], cnt);
  __syncthreads();
  if (tid < qrows && s_cnt[tid]) {
    atomicAdd(P.counts + (q0 + tid) * 4 + P.col, s_cnt[tid]);
    atomicAdd(P.counts + (q0 + tid) * 4 + P.col + 1, s_cnt[tid]);
  }
}

// Two entry points over the same body: ptxas keeps the one-term ops within 128 registers on its
// own (and spills if it is told to), while the two-term dot kernel needs the explicit
// 2-CTAs-per-SM bound to stop it from hoisting the next operand loads into extra registers.
template <int OP, bool L1>
__global__ void __launch_bounds__(kTThreads)
sweep_tiled_kernel(const __grid_constant__ TiledParams P, const __grid_constant__ TiledMaps TM) {
  sweep_tiled_body<OP, L1>(P, TM, blockIdx.x);
}
template <int OP, bool L1>
__global__ void __launch_bounds__(kTThreads, 2)
sweep_tiled_kernel_2cta(const __grid_constant__ TiledParams P, const __grid_constant__ TiledMaps TM) {
  sweep_tiled_body<OP, L1>(P, TM, blockIdx.x);
}

// The tensor-core path's one launch per direction after the sweep.  The sweep has finished, so the pair list's
// length and overflow flag are final:
//   no overflow: resolve the band pairs (into tc_counts) and the filter entries; the last CTA to finish (fenced
//                done counter ctrl[2], reset for the next call or graph replay) then commits the direction,
//                counts[q][col], counts[q][col + 1] += tc_counts[q];
//   overflow (degenerate tables): the fp32 tiled sweep of the direction, one work unit per CTA, then the filter
//                corrections.
// The fallback is a call of its own: inlined, its register pressure would spill into the resolve loop that
// every call runs.
template <int OP>
__device__ __noinline__ void tiled_fallback(const TiledParams& P, const TiledMaps& TM, int unit) {
  sweep_tiled_body<OP, false>(P, TM, unit);
}

// (2 CTAs per SM, as the resolve kernel of the gather and fp32 paths and the tiled sweep run: 128 registers)
template <int MODEL, int VEC, int GROUPING, int OP>
__global__ void __launch_bounds__(kTThreads, 2)
tc_resolve_commit_kernel(const __grid_constant__ ModelParams MP, const __grid_constant__ ResolveArgs A,
                         const __grid_constant__ TiledParams TP, const __grid_constant__ TiledMaps TM) {
  extern __shared__ float4 smem_f4[];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * A.scratch_floats;
  const unsigned listed = *reinterpret_cast<const volatile unsigned*>(A.ctrl);
  const bool overflow = listed > A.cap || *reinterpret_cast<const volatile unsigned*>(A.ctrl + 1) != 0u;
  if (overflow) {
    if ((int)blockIdx.x < TP.units) tiled_fallback<OP>(TP, TM, blockIdx.x);
    __syncthreads();   // the sweep's shared memory becomes the group scratch
    resolve_items<MODEL, VEC, GROUPING>(MP, A, 0, scratch);
    return;
  }
  resolve_items<MODEL, VEC, GROUPING>(MP, A, (int64_t)listed, scratch);
  __threadfence();     // every thread's tc_counts updates, then the whole CTA, before its arrival on the done counter
  __syncthreads();
  unsigned prev = 0u;
  if (threadIdx.x == 0) prev = atomicAdd(A.ctrl + 2, 1u);
  if (!__syncthreads_or(threadIdx.x == 0 && prev == gridDim.x - 1)) return;
  __threadfence();
  for (int64_t q = threadIdx.x; q < A.Q; q += blockDim.x) {
    const int c = __ldcg(A.tc_counts + q);
    if (c) { atomicAdd(A.counts + q * 4 + A.col, c); atomicAdd(A.counts + q * 4 + A.col + 1, c); }
  }
  if (threadIdx.x == 0) A.ctrl[2] = 0u;
}

// ---- preparation kernels -------------------------------------------------------------------------
// query vectors [Q][KQ][dp] (zero padded) + qscale; one 8-lane group per query
template <int MODEL, int VEC, int DIR>
__global__ void __launch_bounds__(256)
prep_query_kernel(ModelParams P, const int64_t* __restrict__ qh, const int64_t* __restrict__ qr,
                  const int64_t* __restrict__ qt, int64_t Q, int dp, float* __restrict__ qvec,
                  float* __restrict__ qscale, float* __restrict__ thr, int scratch_floats, const TcQueryArgs TC) {
  extern __shared__ float4 smem_f4[];
  float* scratch = reinterpret_cast<float*>(smem_f4) + (size_t)(threadIdx.x >> 3) * scratch_floats;
  const int lane = threadIdx.x & 7;
  const int64_t q = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  if (TC.A0 && blockIdx.x == 0 && threadIdx.x < 4) TC.ctrl[threadIdx.x] = 0u;   // pair-list length, overflow, done counter (+ 1 unused)
  if (q >= Q) return;
  const int d = P.d, nch = (d + 3) >> 2, nchp = dp >> 2;
  TripleRows R;
  resolve_rows<MODEL>(R, P, P.qtab, P.qtab, P.qtab, __ldg(qh + q), __ldg(qr + q), __ldg(qt + q));
  prefetch_triple_rows(R, P.d, P.dr, lane);
  // threshold = the target's own score in this direction's grouping (== kge_score_fwd)
  const float s_target = score_group<MODEL, VEC, DIR == 0 ? KGE_GROUP_TAIL : KGE_GROUP_HEAD>(R, P, lane, scratch);
  if (lane == 0) thr[q] = s_target;
  constexpr int KQ = rank_kq(MODEL);
  float* out = qvec + (size_t)q * KQ * dp;
  auto st = [&](int k, int c, float4 v) { *reinterpret_cast<float4*>(out + (size_t)k * dp + 4 * c) = v; };
  const float4 zero = make_float4(0.f, 0.f, 0.f, 0.f);
  if (MODEL == KGE_TRANSE || MODEL == KGE_TRANSM) {
    const float* a = (DIR == 0) ? R.h[0] : R.r[0];   // TAIL: h^ + r^ ; HEAD: r^ - t^
    const float* b = (DIR == 0) ? R.r[0] : R.t[0];
    float sa = 0.f, sb = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 x = ld_chunk<VEC>(a, c, d), y = ld_chunk<VEC>(b, c, d);
#pragma unroll
      for (int e = 0; e < 4; ++e) { sa = ffma(f4_get(x, e), f4_get(x, e), sa); sb = ffma(f4_get(y, e), f4_get(y, e), sb); }
    }
    const float ia = inv_norm_from_sumsq(group_sum(sa)), ib = inv_norm_from_sumsq(group_sum(sb));
    for (int c = lane; c < nchp; c += 8) {
      float4 o = zero;
      if (c < nch) {
        const float4 x = ld_chunk<VEC>(a, c, d), y = ld_chunk<VEC>(b, c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float xn = fmul(f4_get(x, e), ia), yn = fmul(f4_get(y, e), ib);
          f4_at(o, e) = (DIR == 0) ? fadd(xn, yn) : fsub(xn, yn);
        }
      }
      st(0, c, o);
    }
    if (MODEL == KGE_TRANSM && lane == 0) qscale[q] = __ldg(R.r[1]);
  } else if (MODEL == KGE_DISTMULT || MODEL == KGE_CP) {
    const float* a = (DIR == 0) ? R.h[0] : R.r[0];   // TAIL: h*r ; HEAD: r*t
    const float* b = (DIR == 0) ? R.r[0] : R.t[0];
    for (int c = lane; c < nchp; c += 8) {
      float4 o = zero;
      if (c < nch) {
        const float4 x = ld_chunk<VEC>(a, c, d), y = ld_chunk<VEC>(b, c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) f4_at(o, e) = fmul(f4_get(x, e), f4_get(y, e));
      }
      st(0, c, o);
    }
  } else if (MODEL == KGE_COMPLEX) {
    const float* er = (DIR == 0) ? R.h[0] : R.t[0];
    const float* ei = (DIR == 0) ? R.h[1] : R.t[1];
    for (int c = lane; c < nchp; c += 8) {
      float4 o0 = zero, o1 = zero;
      if (c < nch) {
        const float4 xr = ld_chunk<VEC>(er, c, d), xi = ld_chunk<VEC>(ei, c, d),
                     rr = ld_chunk<VEC>(R.r[0], c, d), ri = ld_chunk<VEC>(R.r[1], c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          if (DIR == 0) {
            f4_at(o0, e) = ffma(f4_get(xr, e), f4_get(rr, e), -fmul(f4_get(xi, e), f4_get(ri, e)));
            f4_at(o1, e) = ffma(f4_get(xi, e), f4_get(rr, e), fmul(f4_get(xr, e), f4_get(ri, e)));
          } else {
            f4_at(o0, e) = ffma(f4_get(xr, e), f4_get(rr, e), fmul(f4_get(xi, e), f4_get(ri, e)));
            f4_at(o1, e) = ffma(f4_get(xi, e), f4_get(rr, e), -fmul(f4_get(xr, e), f4_get(ri, e)));
          }
        }
      }
      st(0, c, o0); st(1, c, o1);
    }
  } else if (MODEL == KGE_HOLE || MODEL == KGE_RESCAL) {
    // score_group left the query-side vector in the group's scratch (HoLE: g at scratch+2*dp,
    // RESCAL: v at scratch); entries beyond d are zero.
    const float* src = (MODEL == KGE_HOLE) ? scratch + 2 * (nch * 4) : scratch;
    for (int c = lane; c < nchp; c += 8) st(0, c, c < nch ? *reinterpret_cast<const float4*>(src + 4 * c) : zero);
  } else if (MODEL == KGE_SIMPLE || MODEL == KGE_SIMPLE_IGNR) {
    const float half = (MODEL == KGE_SIMPLE) ? 0.5f : 1.0f;
    for (int c = lane; c < nchp; c += 8) {
      float4 o0 = zero, o1 = zero;
      if (c < nch) {
        const float4 r1 = ld_chunk<VEC>(R.r[0], c, d), r2 = ld_chunk<VEC>(R.r[1], c, d);
        // TAIL: q1 = h1 r1, q2 = half t2 r2 ; HEAD: q1 = r1 t1, q2 = half r2 h2
        const float4 a = ld_chunk<VEC>(DIR == 0 ? R.h[0] : R.t[0], c, d);
        const float4 b = ld_chunk<VEC>(DIR == 0 ? R.h[1] : R.t[1], c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          f4_at(o0, e) = fmul(f4_get(a, e), f4_get(r1, e));
          f4_at(o1, e) = fmul(fmul(f4_get(b, e), f4_get(r2, e)), half);
        }
      }
      st(0, c, o0); st(1, c, o1);
    }
  } else if (MODEL == KGE_ROTATE) {
    // TAIL: q = h o r ; HEAD: q = t o conj(r)  (|h o r - t| = |h - t o conj(r)| for the unit rotation;
    // each grouping is its own canonical arithmetic, DESIGN.md §3 rule 5)
    const float* er = (DIR == 0) ? R.h[0] : R.t[0];
    const float* ei = (DIR == 0) ? R.h[1] : R.t[1];
    for (int c = lane; c < nchp; c += 8) {
      float4 o0 = zero, o1 = zero;
      if (c < nch) {
        const float4 rr = ld_chunk<VEC>(R.r[0], c, d), xr = ld_chunk<VEC>(er, c, d), xi = ld_chunk<VEC>(ei, c, d);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          float im, re;
          sincos_canon(fmul(f4_get(rr, e), P.phase), im, re);
          rot_query(f4_get(xr, e), f4_get(xi, e), re, im, DIR == 1, f4_at(o0, e), f4_at(o1, e));
        }
      }
      st(0, c, o0); st(1, c, o1);
    }
  }
  if (TC.A0) {
    // tensor-core level: bf16 split of the vectors just written (a lane reads chunks other lanes of its
    // group stored: order the group's global writes first) + the accumulator thresholds
    __syncwarp(group_mask());
    tc_query_finish(TC, out, s_target, q, lane, KQ * dp);
  }
}

// candidate scratch: row e -> (normalised | copied) and zero padded to dp
// HoLE candidates: even part of every row (see even_chunk)
__global__ void __launch_bounds__(256)
prep_cand_even_kernel(const float* __restrict__ table, int64_t nc, int d, int dp, float* __restrict__ out) {
  const int lane = threadIdx.x & 7;
  const int64_t e = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  if (e >= nc) return;
  const float* row = table + (size_t)e * d;
  const int nch = (d + 3) >> 2, nchp = dp >> 2;
  for (int c = lane; c < nchp; c += 8)
    *reinterpret_cast<float4*>(out + (size_t)e * dp + 4 * c) =
        c < nch ? even_chunk(row, c, d) : make_float4(0.f, 0.f, 0.f, 0.f);
}

template <int VEC, bool NORMALISE>
__global__ void __launch_bounds__(256)
prep_cand_kernel(const float* __restrict__ table, int64_t nc, int d, int dp, float* __restrict__ out) {
  const int lane = threadIdx.x & 7;
  const int64_t e = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  if (e >= nc) return;
  const float* row = table + (size_t)e * d;
  const int nch = (d + 3) >> 2, nchp = dp >> 2;
  float inv = 1.f;
  if (NORMALISE) {
    float s = 0.f;
    for (int c = lane; c < nch; c += 8) {
      const float4 x = ld_chunk<VEC>(row, c, d);
#pragma unroll
      for (int k = 0; k < 4; ++k) s = ffma(f4_get(x, k), f4_get(x, k), s);
    }
    inv = inv_norm_from_sumsq(group_sum(s));
  }
  for (int c = lane; c < nchp; c += 8) {
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (c < nch) {
      o = ld_chunk<VEC>(row, c, d);
      if (NORMALISE) { o.x = fmul(o.x, inv); o.y = fmul(o.y, inv); o.z = fmul(o.z, inv); o.w = fmul(o.w, inv); }
    }
    *reinterpret_cast<float4*>(out + (size_t)e * dp + 4 * c) = o;
  }
}

int model_vec(const kge_model_t* m);

// candidate source tables of a sweep direction; returns true when a scratch copy is needed
// (normalised rows for TransE/TransM, padding for d % 4 != 0, unaligned tables)
static bool cand_sources(const kge_model_t* m, int dir, const float* src[2]) {
  const int KC = rank_kq(m->model);
  src[0] = src[1] = nullptr;
  if (m->model == KGE_CP) src[0] = m->tables[dir == 0 ? 2 : 0];
  else if (is_simple(m->model)) {  // TAIL: (t1, h2) = (ent_tail, ent_head)[c]; HEAD: (h1, t2) = (ent_head, ent_tail)[c]
    src[0] = m->tables[dir == 0 ? 1 : 0]; src[1] = m->tables[dir == 0 ? 0 : 1];
  } else { src[0] = m->tables[0]; if (KC == 2) src[1] = m->tables[1]; }
  bool scratch = (m->model == KGE_TRANSE || m->model == KGE_TRANSM || m->model == KGE_HOLE) || (m->dim % 4 != 0);
  for (int k = 0; k < KC; ++k) if ((uintptr_t)src[k] & 15) scratch = true;
  return scratch;
}

static int fill_cand_scratch(const RankCall& C, const float* const src[2], cudaStream_t st) {
  const kge_model_t* m = C.m;
  const int KC = rank_kq(m->model), d = m->dim, dp = rank_dp(m);
  const bool normalise = (m->model == KGE_TRANSE || m->model == KGE_TRANSM);
  const int vc = pick_vec(src, KC, d);
  auto kernel = vc == 4 ? (normalise ? prep_cand_kernel<4, true> : prep_cand_kernel<4, false>)
              : vc == 2 ? (normalise ? prep_cand_kernel<2, true> : prep_cand_kernel<2, false>)
                        : (normalise ? prep_cand_kernel<1, true> : prep_cand_kernel<1, false>);
  if (m->model == KGE_HOLE) kernel = prep_cand_even_kernel;
  for (int k = 0; k < KC; ++k) {
    kernel<<<(unsigned)((C.nc + 31) / 32), 256, 0, st>>>(src[k], C.nc, d, dp, C.at<float>(C.L.cand) + (size_t)k * (size_t)C.nc * dp);
    KGE_CHECK_LAUNCH("prep_cand_kernel");
  }
  return KGE_OK;
}

// TransE on the tensor-core path: when TMA can read the table itself (rows of whole 16-byte chunks, 16-byte
// aligned), the fp32 fallback stages the raw rows and normalises them in shared memory with the inverse norms
// tc_prep_cand_kernel writes, instead of reading a normalised scratch copy that the usual call never needs
static bool tc_raw_transe(const RankCall& C) {
  return C.use_tc && C.m->model == KGE_TRANSE && C.m->dim % 4 == 0 && ((uintptr_t)C.m->tables[0] & 15) == 0;
}

int prepare_candidates(const RankCall& C, cudaStream_t st) {
  if (C.m->model == KGE_CP || is_simple(C.m->model)) return KGE_OK;  // per direction: prepare_queries / tiled_sweep
  const float* src[2];
  const bool scratch = cand_sources(C.m, 0, src);
  if (C.use_tc) {  // one kernel: bf16 split for the tensor cores + what the fp32 fallback needs, if anything
    if (tc_raw_transe(C)) return tc_prepare_candidates(C, src, nullptr, C.at<float>(C.L.cinv), st);
    return tc_prepare_candidates(C, src, scratch ? C.at<float>(C.L.cand) : nullptr, nullptr, st);
  }
  if (scratch) return fill_cand_scratch(C, src, st);
  return KGE_OK;
}

bool tiled_supported(const kge_model_t* m) {
  switch (m->model) {
    case KGE_TRANSE: case KGE_TRANSM: case KGE_DISTMULT: case KGE_CP: case KGE_COMPLEX: case KGE_ROTATE:
    case KGE_HOLE: case KGE_RESCAL: case KGE_SIMPLE: case KGE_SIMPLE_IGNR:
      return true;
    default: return false;
  }
}

int prepare_queries(const RankCall& C, int dir, cudaStream_t st) {
  const kge_model_t* m = C.m;
  // CP sweeps the object table for tails and the subject table for heads: its tensor-core candidate
  // operands are per direction and come first
  if (m->model == KGE_CP && C.use_tc) {
    const float* src[2] = {nullptr, nullptr};
    const bool scratch = cand_sources(m, dir, src);
    const int rc = tc_prepare_candidates(C, src, scratch ? C.at<float>(C.L.cand) : nullptr, nullptr, st);
    if (rc) return rc;
  }
  // query vectors and thresholds from the query-side tables
  const ModelParams PQ = make_params(C.mq, C.mq);
  const int vq = model_vec(C.mq);
  const int psf = (int)group_scratch_floats(C.mq);
  const size_t psmem = (size_t)psf * 32 * sizeof(float);
  TcQueryArgs TCQ;
  TCQ.A0 = nullptr;
  if (C.use_tc) TCQ = tc_query_args(C, dir);
  decltype(&prep_query_kernel<KGE_TRANSE, 4, 0>) kernel;
#define PICK(M, V) kernel = dir == 0 ? prep_query_kernel<M, V, 0> : prep_query_kernel<M, V, 1>
  switch (m->model) {
    case KGE_HOLE: KGE_DISPATCH_VEC(KGE_HOLE, vq, PICK); break;
    case KGE_RESCAL: KGE_DISPATCH_VEC(KGE_RESCAL, vq, PICK); break;
    case KGE_SIMPLE: KGE_DISPATCH_VEC(KGE_SIMPLE, vq, PICK); break;
    case KGE_SIMPLE_IGNR: KGE_DISPATCH_VEC(KGE_SIMPLE_IGNR, vq, PICK); break;
    case KGE_TRANSE: KGE_DISPATCH_VEC(KGE_TRANSE, vq, PICK); break;
    case KGE_TRANSM: KGE_DISPATCH_VEC(KGE_TRANSM, vq, PICK); break;
    case KGE_DISTMULT: KGE_DISPATCH_VEC(KGE_DISTMULT, vq, PICK); break;
    case KGE_CP: KGE_DISPATCH_VEC(KGE_CP, vq, PICK); break;
    case KGE_COMPLEX: KGE_DISPATCH_VEC(KGE_COMPLEX, vq, PICK); break;
    default: KGE_DISPATCH_VEC(KGE_ROTATE, vq, PICK); break;
  }
#undef PICK
  const int rc = smem_optin(kernel, psmem);
  if (rc) return rc;
  kernel<<<(unsigned)((C.Q + 31) / 32), 256, psmem, st>>>(PQ, C.qh, C.qr, C.qt, C.Q, rank_dp(m), C.at<float>(C.L.qvec[dir]),
                                                           C.at<float>(C.L.qscale[dir]), C.thr(dir), psf, TCQ);
  KGE_CHECK_LAUNCH("prep_query_kernel");
  return KGE_OK;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
int make_tensor_map(CUtensorMap* tm, CUtensorMapDataType dtype, const void* base, uint64_t rows, uint64_t cols,
                    uint64_t pitch_bytes, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle) {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
    if (!fn) { set_error("cuTensorMapEncodeTiled is not available"); return KGE_ECUDA; }
  }
  const cuuint64_t gdim[2] = {cols, rows};
  const cuuint64_t gstride[1] = {pitch_bytes};
  const cuuint32_t box[2] = {box_cols, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = fn(tm, dtype, 2, const_cast<void*>(base), gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return KGE_ECUDA; }
  return KGE_OK;
}

// One direction's fp32 tiled sweep: parameters, tensor maps and launch shape (a 1-D grid of P.units CTAs).
struct TiledPlan { TiledParams P; TiledMaps TM; size_t smem; int op; };

static int tiled_plan(const RankCall& C, int dir, cudaStream_t st, TiledPlan& T) {
  const kge_model_t* m = C.m;
  const int model = m->model, dp = rank_dp(m), KQ = rank_kq(model), KC = KQ;
  const int64_t Q = C.Q, nc = C.nc;
  T.op = (model == KGE_TRANSE || model == KGE_TRANSM) ? (dir == 0 ? OP_TRANS_T : OP_TRANS_H)
       : (model == KGE_DISTMULT || model == KGE_CP || model == KGE_HOLE || model == KGE_RESCAL) ? OP_DOT1
       : (model == KGE_COMPLEX || is_simple(model)) ? OP_DOT2 : OP_ROT;
  const int TQ = 4;
  const int QBLK = kGQ * TQ;
  TiledParams& P = T.P;

  // candidate arrays: the model's tables, or the scratch copy (made by prepare_candidates, or filled here
  // when the tables differ per direction)
  P.cand_inv = nullptr;
  {
    const float* src[2] = {nullptr, nullptr};
    float* cscratch = C.at<float>(C.L.cand);
    const bool scratch = cand_sources(m, dir, src);
    if (tc_raw_transe(C)) {
      P.cand[0] = src[0]; P.cand[1] = nullptr; P.cand_pitch = m->dim;
      P.cand_inv = C.at<float>(C.L.cinv);
    } else if (scratch) {
      for (int k = 0; k < KC; ++k) P.cand[k] = cscratch + (size_t)k * (size_t)nc * dp;
      if (KC == 1) P.cand[1] = nullptr;
      P.cand_pitch = dp;
      if ((model == KGE_CP && !C.use_tc) || is_simple(model)) {
        const int rc = fill_cand_scratch(C, src, st);
        if (rc) return rc;
      }
    } else {
      P.cand[0] = src[0]; P.cand[1] = src[1]; P.cand_pitch = m->dim;
    }
  }

  // shared-memory plan (DS = columns staged per iteration, a multiple of 32 = whole octets):
  // whole rows when two CTAs of them fit in one SM (228 KB minus 1 KB reserved per CTA), else
  // slabs of DS columns with the accumulators living across slabs
  const size_t budget = (228 * 1024) / 2 - 1024;
  const size_t hdr = (32 + 3 * (size_t)QBLK * 4 + 127) / 128 * 128;
  auto bytes_for = [&](int DS, int qstages) {
    return hdr + ((size_t)QBLK * KQ * qstages + (size_t)kCBLK * KC * 2) * (size_t)DS * sizeof(float);
  };
  const int dp32 = (dp + 31) / 32 * 32;
  int DS, nslabs;
  if (dp32 <= 256 && bytes_for(dp32, 1) <= budget) { DS = dp32; nslabs = 1; }
  else {
    DS = 32;
    while (DS + 32 <= dp32 && DS + 32 <= 256 && bytes_for(DS + 32, 2) <= budget) DS += 32;
    nslabs = (dp + DS - 1) / DS;
  }
  T.smem = bytes_for(DS, nslabs > 1 ? 2 : 1);
  P.qvec = C.at<float>(C.L.qvec[dir]); P.thr = C.thr(dir);
  P.qscale = (model == KGE_TRANSM) ? C.at<float>(C.L.qscale[dir]) : nullptr;
  P.Q = Q; P.nc = nc; P.dp = dp; P.DS = DS; P.nslabs = nslabs;
  P.ntiles = (int)((nc + kCBLK - 1) / kCBLK);
  const int qblocks = (int)((Q + QBLK - 1) / QBLK);
  const int ctas_per_sm = (T.smem + 1024) * 2 <= 228 * 1024 ? 2 : 1;
  int splits = (sm_count() * ctas_per_sm + qblocks - 1) / qblocks;
  if (splits < 1) splits = 1;
  if (splits > P.ntiles) splits = P.ntiles;
  P.tiles_per_cta = (P.ntiles + splits - 1) / splits;
  splits = (P.ntiles + P.tiles_per_cta - 1) / P.tiles_per_cta;
  P.splits = splits; P.units = splits * qblocks;
  P.counts = C.counts; P.col = 2 * dir; P.l1 = m->l1_flag; P.margin = m->margin;
  P.fin = (model == KGE_HOLE) ? 1 : (is_simple(model) ? 2 : 0);

  // fp32 matrices; one box = one octet: 32 columns x all rows of the tile (columns >= dp / rows >= extent read as zeros)
  auto map = [&](CUtensorMap* tm, const float* base, uint64_t rows, uint64_t pitch, uint32_t box_rows) {
    return make_tensor_map(tm, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, base, rows, (uint64_t)P.dp, pitch * sizeof(float), 32u,
                           box_rows, CU_TENSOR_MAP_SWIZZLE_NONE);
  };
  int rc = map(&T.TM.q, P.qvec, (uint64_t)P.Q * KQ, (uint64_t)P.dp, (uint32_t)(QBLK * KQ));
  if (rc) return rc;
  rc = map(&T.TM.c0, P.cand[0], (uint64_t)P.nc, (uint64_t)P.cand_pitch, (uint32_t)kCBLK);
  if (rc) return rc;
  T.TM.c1 = T.TM.c0;
  if (KC == 2) {
    rc = map(&T.TM.c1, P.cand[1], (uint64_t)P.nc, (uint64_t)P.cand_pitch, (uint32_t)kCBLK);
    if (rc) return rc;
  }
  return KGE_OK;
}

template <int OP, bool L1>
static int launch_sweep(const TiledPlan& T, SweepProfile* prof, cudaStream_t st) {
  const auto kernel = [] {
    if constexpr (OP == OP_DOT2) return sweep_tiled_kernel_2cta<OP, L1>;
    else return sweep_tiled_kernel<OP, L1>;
  }();
  const int rc = smem_optin(kernel, T.smem);
  if (rc) return rc;
  if (prof) KGE_CUDA_OK(cudaEventRecord(prof->beg, st));
  kernel<<<(unsigned)T.P.units, kTThreads, T.smem, st>>>(T.P, T.TM);
  KGE_CHECK_LAUNCH("sweep_tiled_kernel");
  if (prof) { KGE_CUDA_OK(cudaEventRecord(prof->end, st)); prof->valid = true; }
  return KGE_OK;
}

int tiled_sweep(const RankCall& C, int dir, cudaStream_t st) {
  TiledPlan T;
  const int rc = tiled_plan(C, dir, st, T);
  if (rc) return rc;
  SweepProfile* prof = sweep_profile(dir)->armed ? sweep_profile(dir) : nullptr;
  const bool l1 = C.m->l1_flag != 0;
  switch (T.op) {
    case OP_TRANS_T: return l1 ? launch_sweep<OP_TRANS_T, true>(T, prof, st) : launch_sweep<OP_TRANS_T, false>(T, prof, st);
    case OP_TRANS_H: return l1 ? launch_sweep<OP_TRANS_H, true>(T, prof, st) : launch_sweep<OP_TRANS_H, false>(T, prof, st);
    case OP_DOT1: return launch_sweep<OP_DOT1, false>(T, prof, st);
    case OP_DOT2: return launch_sweep<OP_DOT2, false>(T, prof, st);
    default: return launch_sweep<OP_ROT, false>(T, prof, st);
  }
}

int tc_resolve_commit(const RankCall& C, int dir, cudaStream_t st) {
  TiledPlan T;
  int rc = tiled_plan(C, dir, st, T);
  if (rc) return rc;
  const GroupArgs G = group_args(C);
  decltype(&tc_resolve_commit_kernel<KGE_TRANSE, 4, KGE_GROUP_TAIL, OP_TRANS_T>) kernel;
#define PICK_OP(M, V, OP) kernel = dir == 0 ? tc_resolve_commit_kernel<M, V, KGE_GROUP_TAIL, OP> \
                                            : tc_resolve_commit_kernel<M, V, KGE_GROUP_HEAD, OP>
#define PICK_TRANSE(M, V) kernel = dir == 0 ? tc_resolve_commit_kernel<M, V, KGE_GROUP_TAIL, OP_TRANS_T> \
                                            : tc_resolve_commit_kernel<M, V, KGE_GROUP_HEAD, OP_TRANS_H>
#define PICK_DOT1(M, V) PICK_OP(M, V, OP_DOT1)
#define PICK_DOT2(M, V) PICK_OP(M, V, OP_DOT2)
#define PICK_ROT(M, V) PICK_OP(M, V, OP_ROT)
  switch (C.m->model) {   // the models tc_supported admits
    case KGE_TRANSE: KGE_DISPATCH_VEC(KGE_TRANSE, G.vec, PICK_TRANSE); break;
    case KGE_DISTMULT: KGE_DISPATCH_VEC(KGE_DISTMULT, G.vec, PICK_DOT1); break;
    case KGE_CP: KGE_DISPATCH_VEC(KGE_CP, G.vec, PICK_DOT1); break;
    case KGE_RESCAL: KGE_DISPATCH_VEC(KGE_RESCAL, G.vec, PICK_DOT1); break;
    case KGE_COMPLEX: KGE_DISPATCH_VEC(KGE_COMPLEX, G.vec, PICK_DOT2); break;
    case KGE_ROTATE: KGE_DISPATCH_VEC(KGE_ROTATE, G.vec, PICK_ROT); break;
    default: set_error("tc_resolve_commit: model %d has no tensor-core path", (int)C.m->model); return KGE_ENOTSUP;
  }
#undef PICK_ROT
#undef PICK_DOT2
#undef PICK_DOT1
#undef PICK_TRANSE
#undef PICK_OP
  const size_t smem = T.smem > G.smem ? T.smem : G.smem;
  rc = smem_optin(kernel, smem);
  if (rc) return rc;
  // band pairs and filter entries grid-stride over two CTAs per SM; the fallback needs one CTA per work unit
  const int grid = T.P.units > 2 * sm_count() ? T.P.units : 2 * sm_count();
  kernel<<<(unsigned)grid, kTThreads, smem, st>>>(G.P, resolve_args(C, dir), T.P, T.TM);
  KGE_CHECK_LAUNCH("tc_resolve_commit_kernel");
  return KGE_OK;
}

}  // namespace kge
