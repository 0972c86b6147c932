// kge_rank_tc.cu — 1-vs-all sweep on the Hopper tensor cores (wgmma + TMA + mbarrier), EXACT.
//
// The batched 1-vs-all sweep of the dot-product / squared-distance models (DistMult, CP, ComplEx,
// RESCAL's h^T M_r . t, TransE-L2, RotatE) is a Q x N x K contraction.  Ranks, however, are
// specified in exact fp32 canonical arithmetic (DESIGN.md §3).  The two are reconciled by a
// TWO-LEVEL comparison instead of trying to make the MMA bit-reproducible:
//
//   level 1 (this file, tensor cores): every fp32 operand x is split into two bf16 terms
//       x0 = bf16_rn(x), x1 = bf16_rn(x - x0)            (|x - x0 - x1| <= 2^-18 |x|)
//     and D(q,c) = sum_k a0 b0 + a0 b1 + a1 b0 is accumulated in fp32 registers by three
//     wgmma.mma_async (m64n128k16, bf16 inputs) per 16-wide k-step and warpgroup; operand tiles arrive
//     by TMA (128-byte swizzle) through a ring of shared-memory stages guarded by mbarriers.
//     Squared distances use |q - c|^2 = |q|^2 - 2 (q.c - |c|^2/2): the candidate norm term rides
//     in three extra k-columns (a 3-way bf16 split of |c|^2/2 against -1), so the epilogue only
//     compares the accumulator with two per-query constants:
//         D > tau_hi[q]  -> the candidate certainly outranks the target (counted here)
//         D < tau_lo[q]  -> it certainly does not
//         otherwise      -> (q, c) is appended to a list
//     tau_hi/lo = centre -+ E with E a PROVEN bound on |D_tc - D_exact| + |canonical fp32 score -
//     exact score| (prep_query below; derivation in DESIGN.md §4b).
//   level 2 (kge_rank.cu, resolve_pairs_kernel): the listed pairs — a handful per query — are
//     re-evaluated with the canonical fp32 group function (the arithmetic of kge_score_fwd /
//     the fp32 sweeps / the CPU oracle) and compared exactly.
//
// The final counts therefore equal the fp32 specification's for every input.  If the list
// overflows (degenerate tables: thousands of exact ties per query) the resolve launch runs the fp32
// tiled sweep of kge_rank_tiled.cu instead, decided on the device (no host sync).
//
// Replaces: Evaluator.test_tail_rank / test_head_rank forward over all N entities + topk
// (pykg2vec/utils/evaluator.py:249-273,309-334) for models pairwise.py:56-93 (TransE, -l1 False),
// :765-791 (RotatE), :829-865 (Rescal), pointwise.py:444-446 (DistMult), :163-188 (Complex),
// :374-376 (CP).
#include <cuda_bf16.h>

#include "kge_models.cuh"
#include "kge_rank.cuh"
#include "kge_rank_tc.cuh"
#include "kge_tma.cuh"

namespace kge {

constexpr int kTcBM = 128;        // queries per CTA: two consumer warpgroups of 64 rows (wgmma M = 64)
constexpr int kTcBN = 128;        // candidates per tile (wgmma N)
constexpr int kTcBK = 64;         // bf16 elements per k-block: one 128-byte swizzle row
constexpr int kTcThreads = 384;   // warpgroup 0: TMA producer (one thread), warpgroups 1-2: wgmma + epilogue
constexpr int kTcConsumerWarps = 8;
constexpr int kTcMaxStages = 8;
constexpr int kTcResidentMaxK = 256;                   // query block stays in smem when Kp <= 256

// The per-direction buffers of a launch: blockIdx.z picks the set (one launch sweeps BOTH directions of a rank
// call — same candidate operands, different query operands — so that the fixed cost of a launch, the pipeline
// ramp and the last tile's drain are paid once, and 2 x qblocks x ntiles tile units balance over the SMs).
struct TcDirView {
  const float* tau;        // [Q][4]: centre, a, b, e (tc_query_finish)
  int32_t* tc_counts;      // [Q]
  unsigned* ctrl;          // [0] list length, [1] overflow ([2] tc_resolve_commit_kernel's done counter)
  unsigned long long* list;
  float* dbg;              // optional [Q][nc] raw accumulators (tests)
};
struct TcParams {
  TcDirView D[2];
  const float* cn;         // [nc] per-candidate norm bound n_c (tc_prep_cand_kernel)
  unsigned cap;
  int64_t Q, nc;
  int Kp, nkb, a_resident, nstages;
  uint32_t tile_bytes;     // one operand k-block tile: 128 rows x kTcBK x 2 bytes
  int tiles_per_cta, ntiles;
  long long* trace;        // optional timeline of CTA (0,0): [3 roles][64] clock64 stamps (kge_debug_set_tc_trace)
};
// a*: query operands of blockIdx.z == 0, c*: of blockIdx.z == 1, b*: candidate operands
struct TcMaps { CUtensorMap a0, a1, b0, b1, c0, c1; };

// ---- wgmma ---------------------------------------------------------------------------------------
// shared-memory matrix descriptor (sm_90 wgmma): K-major operand tile [rows][64 bf16] written by TMA with the
// 128-byte swizzle.  start address >> 4 in bits [0,14); leading byte offset (unused for swizzled K-major,
// canonical value 1) in [16,30); stride byte offset = 8 rows x 128 B = 1024 (>> 4) in [32,46); layout type
// SWIZZLE_128B = 1 in [62,64).  16 bf16 further along k = 32 bytes further along the swizzled row: +2.
KGE_DEV uint64_t tc_smem_desc(uint32_t addr) {
  uint64_t d = 0;
  d |= (uint64_t)((addr >> 4) & 0x3FFF);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024u >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}
KGE_DEV void tc_wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
KGE_DEV void tc_wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
KGE_DEV void tc_wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// d[64] (+)= A[smem, 64 x 16] . B[smem, 128 x 16]^T, bf16 inputs, fp32 accumulate, both operands K-major.
// Fragment of thread (warp w of the warpgroup, lane l): d[4j + 2i + c] = row 16w + l/4 + 8i, column 8j + 2(l%4) + c.
KGE_DEV void tc_wgmma(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
      "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
      "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
      "%64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
        "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
        "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
        "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
        "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
        "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
        "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
        "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

// timeline stamps of CTA (0,0) (measurement aid; P.trace is null in normal operation).  `slot` is evaluated
// once: callers pass counters with side effects (ev++).
#define TC_STAMP(role, slot)                                                                         \
  do {                                                                                               \
    const int tc_slot_ = (slot);                                                                     \
    if (P.trace && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0 && (tc_slot_ < 62 || tc_slot_ == 63)) \
      P.trace[(role) * 64 + tc_slot_] = clock64();                                                   \
  } while (0)

// Pair-list slots are handed out per WARP in blocks (16 slots) reserved with one global atomic (a returning
// atomic per ambiguous pair would stall the epilogue on its round trip): base/size = the warp's current block
// in P.list, used = slots already written.  Unused slots of a block are filled with the sentinel ~0
// (resolve_pairs_kernel skips them), so [0, ctrl[0]) is always fully defined.
struct TcListState { unsigned base, used, size; };
constexpr unsigned long long kTcListHole = ~0ull;
constexpr unsigned kTcListBlock = 16;

KGE_DEV void tc_list_reserve(TcListState& L, const TcParams& P, const TcDirView& V, int lane, unsigned need) {
  unsigned b = 0;
  if (lane == 0) {
    b = atomicAdd(&V.ctrl[0], need);
    if (b + need > P.cap) V.ctrl[1] = 1u;   // overflow: the exact fp32 sweep takes over (list writes are bounded)
  }
  L.base = __shfl_sync(0xffffffffu, b, 0);
  L.used = 0u;
  L.size = need;
}

KGE_DEV void tc_list_pad(TcListState& L, const TcParams& P, const TcDirView& V, int lane) {
  for (unsigned i = L.used + (unsigned)lane; i < L.size; i += 32u)
    if (L.base + i < P.cap) V.list[L.base + i] = kTcListHole;
  L.used = L.size;
}

// The band test of one accumulator: half-width of the pair from the candidate's norm bound (two fma),
// u = D - centre; certainly better when u > half, inside the band when -half <= u <= half.
struct TcBand { float centre, a, b, e; };
KGE_DEV void tc_band_eval(const TcBand& Bq, float x, float n, float& u, float& half) {
  half = __fmaf_rn(__fmaf_rn(Bq.e, n, Bq.b), n, Bq.a);
  u = __fsub_rn(x, Bq.centre);
}

// Epilogue of one 64 x 128 accumulator tile held by a warpgroup: this thread's rows qa (= q of i = 0) and qa + 8,
// columns 8j + 2(lane%4) + c of the tile (cbase + ...).  Counts the certainly-better candidates per row; warps in
// which some pair lies inside its band list those pairs (a warp-level exclusive scan assigns the slots).
// The band test runs once per pair: its in-band outcomes are kept as bits 4j + 2c + i of band[2] (j < 8 in band[0]),
// and the listing walks the set bits — a handful per tile in a warp — instead of re-testing all 64 pairs.
KGE_DEV void tc_epilogue(const float (&acc)[64], const float (&nl)[32], const TcBand (&Bq)[2], int64_t qa, int64_t cbase,
                         int nvalid, const TcParams& P, const TcDirView& V, TcListState& L, int lane, int (&cnt)[2]) {
  const int cl = 2 * (lane & 3);
  unsigned band[2] = {0u, 0u};
#pragma unroll
  for (int j = 0; j < 16; ++j) {
#pragma unroll
    for (int c = 0; c < 2; ++c) {
      const bool ok = 8 * j + cl + c < nvalid;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float u, h;
        tc_band_eval(Bq[i], acc[4 * j + 2 * i + c], nl[2 * j + c], u, h);
        cnt[i] += (ok && u > h) ? 1 : 0;
        band[j >> 3] |= (ok && u >= -h && !(u > h)) ? 1u << ((4 * j + 2 * c + i) & 31) : 0u;
      }
    }
  }
  const int amb = __popc(band[0]) + __popc(band[1]);
  if (__any_sync(0xffffffffu, amb != 0)) {
    int incl = amb;
#pragma unroll
    for (int off = 1; off < 32; off <<= 1) {
      const int t = __shfl_up_sync(0xffffffffu, incl, off);
      if (lane >= off) incl += t;
    }
    const unsigned total = (unsigned)__shfl_sync(0xffffffffu, incl, 31);
    if (L.used + total > L.size) {   // next block (rare: the first block is reserved before the first tile)
      tc_list_pad(L, P, V, lane);
      tc_list_reserve(L, P, V, lane, total > kTcListBlock ? total : kTcListBlock);
    }
    unsigned k = L.base + L.used + (unsigned)(incl - amb);
#pragma unroll
    for (int w = 0; w < 2; ++w) {
      for (unsigned m = band[w]; m != 0u; m &= m - 1u) {   // ascending bits: the order of the pairs is (j, c, i)
        const int b = 32 * w + __ffs(m) - 1;
        const int i = b & 1, col = 8 * (b >> 2) + cl + ((b >> 1) & 1);
        if (k < P.cap) V.list[k] = ((unsigned long long)(qa + 8 * i) << 32) | (unsigned long long)(cbase + col);
        ++k;
      }
    }
    L.used += total;
  }
  if (V.dbg) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t q = qa + 8 * i;
      if (q >= P.Q) continue;
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c)
          if (8 * j + cl + c < nvalid) V.dbg[(size_t)q * (size_t)P.nc + (size_t)(cbase + 8 * j + cl + c)] = acc[4 * j + 2 * i + c];
    }
  }
}

// ---- the sweep ------------------------------------------------------------------------------------
// grid (splits, query blocks, directions); CTA = 128 queries x a run of 128-candidate tiles.
//   warpgroup 0, thread 0 : TMA producer (query k-blocks once when they fit, riding on the first tile's
//                           stages; candidate k-blocks — and streamed query k-blocks — through a ring of stages)
//   warpgroups 1, 2       : query rows [0, 64) / [64, 128) of the block.  Per k-block 3 x (Kp/16 per block)
//                           wgmma into 64 fp32 registers per thread; a stage is released (one arrive per warp on
//                           its empty barrier) once the wgmma group that read it has retired; after the tile's
//                           last k-block the warpgroup runs the band epilogue on its registers while the producer
//                           keeps filling stages for the next tile.
__global__ void __launch_bounds__(kTcThreads, 1)
tc_sweep_kernel(const __grid_constant__ TcParams P, const __grid_constant__ TcMaps TM) {
  extern __shared__ unsigned char tc_smem_raw[];
  const int t0 = blockIdx.x * P.tiles_per_cta;
  const int ntl = min(P.tiles_per_cta, P.ntiles - t0);
  if (ntl <= 0) return;
  const uint32_t raw = smem_u32(tc_smem_raw);
  const uint32_t base = (raw + 1023u) & ~1023u;                 // SWIZZLE_128B tiles need 1024-byte alignment
  unsigned char* const gbase = tc_smem_raw + (base - raw);
  uint64_t* const full = reinterpret_cast<uint64_t*>(gbase);    // control block: first 1024 bytes
  uint64_t* const empty = full + kTcMaxStages;
  const uint32_t a_base = base + 1024u;                         // resident query k-blocks
  const uint32_t tb = P.tile_bytes;
  const uint32_t a_bytes = P.a_resident ? (uint32_t)P.nkb * 2u * tb : 0u;
  const uint32_t st_base = a_base + a_bytes;
  const uint32_t st_bytes = (P.a_resident ? 2u : 4u) * tb;     // [B0][B1]([A0][A1])

  const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int64_t q0 = (int64_t)blockIdx.y * kTcBM;
  const bool zdir = blockIdx.z != 0;
  const TcDirView& V = zdir ? P.D[1] : P.D[0];
  const CUtensorMap* const ma0 = zdir ? &TM.c0 : &TM.a0;
  const CUtensorMap* const ma1 = zdir ? &TM.c1 : &TM.a1;
  if (threadIdx.x == 0) TC_STAMP(2, 63);   // kernel entry of CTA (0,0)
  // wall-clock span of EVERY CTA (%globaltimer, ns) behind the three role timelines: launch skew and stragglers
  const unsigned cta_lin = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
  if (P.trace && threadIdx.x == 0 && cta_lin < 1024u) {
    unsigned long long ns;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
    P.trace[192 + 2 * cta_lin] = (long long)ns;
  }

  if (threadIdx.x == 0) {
    for (int s = 0; s < P.nstages; ++s) { mbar_init(&full[s], 1); mbar_init(&empty[s], kTcConsumerWarps); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (wg == 0) {
    // the producer needs few registers: hand them to the consumers' 64 accumulators + 32 norm bounds
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;" ::: "memory");
    if (threadIdx.x == 0) {
      int stage = 0; uint32_t phase = 0;
      int ev = 0;
      TC_STAMP(0, ev++);
      for (int t = 0; t < ntl; ++t) {
        const int row = (t0 + t) * kTcBN;
        for (int kb = 0; kb < P.nkb; ++kb) {
          mbar_wait(&empty[stage], phase ^ 1u);
          TC_STAMP(0, ev++);
          // resident query k-blocks ride on the FIRST tile's stage barriers, k-block by k-block: the first wgmma
          // needs one k-block of each operand in shared memory, not the whole query block
          const bool with_a = P.a_resident && t == 0;
          mbar_arrive_expect_tx(&full[stage], ((P.a_resident && !with_a) ? 2u : 4u) * tb);
          const uint32_t sb = st_base + (uint32_t)stage * st_bytes;
          const int col = kb * kTcBK;
          if (with_a) {
            const uint32_t dst = a_base + (uint32_t)kb * 2u * tb;
            tma_load_2d(dst, ma0, col, (int)q0, &full[stage]);
            tma_load_2d(dst + tb, ma1, col, (int)q0, &full[stage]);
          }
          tma_load_2d(sb, &TM.b0, col, row, &full[stage]);
          tma_load_2d(sb + tb, &TM.b1, col, row, &full[stage]);
          if (!P.a_resident) {
            tma_load_2d(sb + 2u * tb, ma0, col, (int)q0, &full[stage]);
            tma_load_2d(sb + 3u * tb, ma1, col, (int)q0, &full[stage]);
          }
          if (++stage == P.nstages) { stage = 0; phase ^= 1u; }
        }
      }
    }
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 232;" ::: "memory");
    const int half = wg - 1;                               // query rows [64 half, 64 half + 64) of the block
    const int64_t qa = q0 + 64 * half + 16 * (warp & 3) + (lane >> 2);   // this thread's rows: qa, qa + 8
    TcBand Bq[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int64_t q = qa + 8 * i;
      Bq[i] = {INFINITY, 0.f, 0.f, 0.f};                   // rows beyond Q: u = -inf -> nothing counted, nothing listed
      if (q < P.Q) {
        const float4 tq = __ldg(reinterpret_cast<const float4*>(V.tau) + q);
        Bq[i] = {tq.x, tq.y, tq.z, tq.w};
      }
    }
    const uint32_t a_off = (uint32_t)half * 64u * (uint32_t)(kTcBK * 2);   // 64 rows of 128 bytes into the A tile
    int cnt[2] = {0, 0};
    TcListState L = {0u, 0u, 0u};
    tc_list_reserve(L, P, V, lane, kTcListBlock);   // the warp's first block: the atomic's round trip hides behind the first tile's MMAs
    // timeline of CTA (0,0,0), warp 4: role 1 = start, then one stamp after each full-barrier wait (slot 63: the
    // cycles spent inside those waits, i.e. starved of operands); role 2 = epilogue begin / end per tile
    const bool stamper = P.trace && warp == 4 && lane == 0;
    int ev = 0, evf = 1;
    long long starved = 0;
    if (stamper) TC_STAMP(1, ev++);
    int stage = 0; uint32_t phase = 0;
    float acc[64];
#pragma unroll
    for (int i = 0; i < 64; ++i) acc[i] = 0.f;
    float nl[32];
    for (int t = 0; t < ntl; ++t) {
      const int64_t cbase = (int64_t)(t0 + t) * kTcBN;
      const int nvalid = (int)min((int64_t)kTcBN, P.nc - cbase);
      // the candidates' norm bounds of this thread's 32 columns, requested before the MMAs so that the L2
      // latency is off the path
#pragma unroll
      for (int j = 0; j < 16; ++j)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int col = 8 * j + 2 * (lane & 3) + c;
          nl[2 * j + c] = col < nvalid ? __ldg(P.cn + cbase + col) : 0.f;
        }
      int prev = -1;
      for (int kb = 0; kb < P.nkb; ++kb) {
        const long long tw = stamper ? clock64() : 0;
        mbar_wait(&full[stage], phase);
        if (stamper) { TC_STAMP(1, evf++); starved += clock64() - tw; }
        const uint32_t sb = st_base + (uint32_t)stage * st_bytes;
        const uint32_t a0 = (P.a_resident ? a_base + (uint32_t)kb * 2u * tb : sb + 2u * tb) + a_off;
        const uint64_t da0 = tc_smem_desc(a0), da1 = tc_smem_desc(a0 + tb);
        const uint64_t db0 = tc_smem_desc(sb), db1 = tc_smem_desc(sb + tb);
        const int nks = min(kTcBK / 16, (P.Kp - kb * kTcBK) / 16);   // Kp is a multiple of 16; columns past it are TMA zero fill
        tc_wgmma_fence();
#pragma unroll 1
        for (int k = 0; k < nks; ++k) {
          const uint64_t ko = (uint64_t)(2 * k);
          tc_wgmma(acc, da0 + ko, db0 + ko, (kb | k) != 0 ? 1u : 0u);
          tc_wgmma(acc, da0 + ko, db1 + ko, 1u);
          tc_wgmma(acc, da1 + ko, db0 + ko, 1u);
        }
        tc_wgmma_commit();
        tc_wgmma_wait<1>();   // the group of the previous k-block has retired: its stage may be refilled
        if (prev >= 0) { __syncwarp(); if (lane == 0) mbar_arrive(&empty[prev]); }
        prev = stage;
        if (++stage == P.nstages) { stage = 0; phase ^= 1u; }
      }
      tc_wgmma_wait<0>();
      __syncwarp();
      if (lane == 0) mbar_arrive(&empty[prev]);
      if (stamper) TC_STAMP(2, ev++);
      tc_epilogue(acc, nl, Bq, qa, cbase, nvalid, P, V, L, lane, cnt);
      if (stamper) TC_STAMP(2, ev++);
    }
    if (stamper && blockIdx.x == 0 && blockIdx.y == 0 && blockIdx.z == 0) P.trace[64 + 63] = starved;
    tc_list_pad(L, P, V, lane);   // the unused slots of the warp's last block become holes
#pragma unroll
    for (int i = 0; i < 2; ++i) {   // the four lanes of a row hold its 32 columns each
      cnt[i] += __shfl_xor_sync(0xffffffffu, cnt[i], 1);
      cnt[i] += __shfl_xor_sync(0xffffffffu, cnt[i], 2);
      const int64_t q = qa + 8 * i;
      if ((lane & 3) == 0 && q < P.Q && cnt[i]) atomicAdd(V.tc_counts + q, cnt[i]);
    }
  }
  __syncthreads();
  if (P.trace && threadIdx.x == 0 && cta_lin < 1024u) {
    unsigned long long ns;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(ns));
    P.trace[192 + 2 * cta_lin + 1] = (long long)ns;
    if (cta_lin == 0) P.trace[2 * 64 + 62] = clock64();   // CTA (0,0,0): cycles at exit, next to its ns span
  }
}

// ---- operand preparation --------------------------------------------------------------------------
// One 8-lane group per candidate row, ONE pass over the fp32 table(s) for everything the row needs:
// (NORMALISE: TransE) the canonical row normalisation of the fp32 sweep — same arithmetic as prep_cand_kernel;
// the fp32 fallback gets either its inverse norm (cinv, when it stages the raw table) or the normalised rows
// (s0, a scratch copy) —, the bf16 split of the KC arrays concatenated along k, the three norm columns
// (squared-distance models) and the row's norm bound n_c.  Rows are read with the widest vector the table
// alignment allows; columns d .. dp-1 are zero.
template <int VEC, bool NORMALISE>
__global__ void __launch_bounds__(256)
tc_prep_cand_kernel(const float* __restrict__ c0, const float* __restrict__ c1, int64_t pitch, int64_t nc, int d,
                    int dp, int KC, int Kp, int aug, __nv_bfloat16* __restrict__ B0, __nv_bfloat16* __restrict__ B1,
                    float* __restrict__ cn, float* __restrict__ s0, float* __restrict__ s1, float* __restrict__ cinv) {
  const int lane = threadIdx.x & 7;
  const int64_t e = (int64_t)blockIdx.x * 32 + (threadIdx.x >> 3);
  if (e >= nc) return;
  const int nch = (d + 3) >> 2, nchp = dp >> 2;
  __nv_bfloat16* o0 = B0 + (size_t)e * Kp;
  __nv_bfloat16* o1 = B1 + (size_t)e * Kp;
  double ss = 0.0;
  for (int k = 0; k < KC; ++k) {
    const float* row = (k == 0 ? c0 : c1) + (size_t)e * pitch;
    float* srow = (k == 0 ? s0 : s1);
    if (srow) srow += (size_t)e * dp;
    float inv = 1.f;
    if (NORMALISE) {
      float s = 0.f;
      for (int c = lane; c < nch; c += 8) {
        const float4 x = ld_chunk<VEC>(row, c, d);
#pragma unroll
        for (int j = 0; j < 4; ++j) s = ffma(f4_get(x, j), f4_get(x, j), s);
      }
      inv = inv_norm_from_sumsq(group_sum(s));
      if (cinv && lane == 0) cinv[e] = inv;   // (KC == 1)
    }
    for (int c = lane; c < nchp; c += 8) {
      float4 x = make_float4(0.f, 0.f, 0.f, 0.f);
      if (c < nch) {
        x = ld_chunk<VEC>(row, c, d);
        if (NORMALISE) { x.x = fmul(x.x, inv); x.y = fmul(x.y, inv); x.z = fmul(x.z, inv); x.w = fmul(x.w, inv); }
      }
      if (srow) *reinterpret_cast<float4*>(srow + 4 * c) = x;
#pragma unroll
      for (int j = 0; j < 4; ++j) ss += (double)f4_get(x, j) * (double)f4_get(x, j);
      tc_split_store(o0 + k * dp + 4 * c, o1 + k * dp + 4 * c, x, 1.0f);
    }
  }
  ss = tc_group_sum_d(ss);
  // |c|^2 / 2 = n0 + n1 + n2 (+ <= 2^-26 relative), multiplied by the query's -1 columns
  const float half = (float)(0.5 * ss);
  const __nv_bfloat16 n0 = __float2bfloat16_rn(half);
  const float r1 = __fsub_rn(half, __bfloat162float(n0));
  const __nv_bfloat16 n1 = __float2bfloat16_rn(r1);
  const __nv_bfloat16 n2 = __float2bfloat16_rn(__fsub_rn(r1, __bfloat162float(n1)));
  tc_store_tail(o0, o1, KC * dp, Kp, lane, aug != 0, n0, n1, n2);
  // upper bound of |c| over the row's actual fp32 operands: the n_c of the pair's error budget (tc_query_finish)
  if (lane == 0) cn[e] = __double2float_ru(sqrt(ss) * (1.0 + 1e-7));
}

static long long* g_tc_trace = nullptr;   // device buffer [3][64] or null (measurement aid)
void tc_set_trace(long long* buf) { g_tc_trace = buf; }

// ---- host side ------------------------------------------------------------------------------------
bool tc_supported(const kge_model_t* m, int64_t nc) {
  if (nc < 1024) return false;                      // small tables: the fp32 sweep is launch-latency sized anyway
  if (nc >= ((int64_t)1 << 31)) return false;
  switch (m->model) {
    case KGE_TRANSE: return m->l1_flag == 0;        // L1 distances are not a contraction
    case KGE_DISTMULT: case KGE_CP: case KGE_COMPLEX: case KGE_RESCAL: case KGE_ROTATE: return true;
    default: return false;                          // HoLE / SimplE / TransM: saturating or scaled finalisers
  }
}

// Candidate operands from the model's own fp32 tables src[k] (row pitch m->dim): bf16 split (+ norm
// columns, + the per-row norm bounds) and, when `scratch` is given, the fp32 copy the fp32 fallback sweep reads
// (normalised for TransE, zero padded to dp), or (TransE) when `cinv` is given the rows' inverse norms — all in
// one kernel.
int tc_prepare_candidates(const RankCall& C, const float* const src[2], float* scratch, float* cinv, cudaStream_t st) {
  const kge_model_t* m = C.m;
  const int64_t nc = C.nc;
  const int KC = rank_kq(m->model), d = m->dim, dp = rank_dp(m), Kp = tc_kp(m), aug = tc_kind(m) != 0 ? 1 : 0;
  const int vc = pick_vec(src, KC, d);
  const bool nrm = m->model == KGE_TRANSE;
  auto kernel = vc == 4 ? (nrm ? tc_prep_cand_kernel<4, true> : tc_prep_cand_kernel<4, false>)
              : vc == 2 ? (nrm ? tc_prep_cand_kernel<2, true> : tc_prep_cand_kernel<2, false>)
                        : (nrm ? tc_prep_cand_kernel<1, true> : tc_prep_cand_kernel<1, false>);
  kernel<<<(unsigned)((nc + 31) / 32), 256, 0, st>>>(
      src[0], KC == 2 ? src[1] : src[0], (int64_t)d, nc, d, dp, KC, Kp, aug, C.at<__nv_bfloat16>(C.L.b[0]),
      C.at<__nv_bfloat16>(C.L.b[1]), C.at<float>(C.L.cn), scratch, (scratch && KC == 2) ? scratch + (size_t)nc * dp : nullptr, cinv);
  KGE_CHECK_LAUNCH("tc_prep_cand_kernel");
  return KGE_OK;
}

// Where prep_query_kernel (kge_rank_tiled.cu) leaves the tensor-core operands of direction `dir`.
TcQueryArgs tc_query_args(const RankCall& C, int dir) {
  TcQueryArgs T;
  T.A0 = C.at<__nv_bfloat16>(C.L.a[dir][0]);
  T.A1 = C.at<__nv_bfloat16>(C.L.a[dir][1]);
  T.tau = C.at<float>(C.L.tau[dir]);
  T.tc_counts = C.at<int32_t>(C.L.tc_counts[dir]);
  T.ctrl = C.at<unsigned>(C.L.ctrl[dir]);
  T.Kp = tc_kp(C.m); T.kind = tc_kind(C.m);
  // head sweep of TransE: canonical distance is |c + q| with q = r^ - t^  ->  contract with -q
  T.sign = (C.m->model == KGE_TRANSE && dir == 1) ? -1.0f : 1.0f;
  T.margin = C.m->margin;
  return T;
}

// Level 1 (the query operands and thresholds were written by prep_query_kernel): the tensor-core sweep of
// direction `dir`, or — ndirs == 2, dir == 0 — of both directions in ONE launch (grid.z = 2).  On return (in
// stream order) tc_counts[q] holds the certain counts and list/ctrl the ambiguous pairs of each direction swept.
int tc_sweep(const RankCall& C, int dir, int ndirs, float* dots, cudaStream_t st) {
  const RankLayout& L = C.L;
  const int64_t Q = C.Q, nc = C.nc;
  const int Kp = tc_kp(C.m);
  if (ndirs < 1 || ndirs > 2 || (ndirs == 2 && dir != 0)) { set_error("tc_sweep: bad direction set"); return KGE_EINVAL; }
  const int dz[2] = {dir, ndirs == 2 ? dir + 1 : dir};   // (an unused second set mirrors the first)
  TcParams P;
  for (int z = 0; z < 2; ++z) {
    P.D[z].tau = C.at<float>(L.tau[dz[z]]);
    P.D[z].tc_counts = C.at<int32_t>(L.tc_counts[dz[z]]);
    P.D[z].ctrl = C.at<unsigned>(L.ctrl[dz[z]]);
    P.D[z].list = C.at<unsigned long long>(L.list[dz[z]]);
    P.D[z].dbg = (z == 0) ? dots : nullptr;
  }
  P.cn = C.at<float>(L.cn); P.cap = tc_list_capacity(Q);
  P.tile_bytes = (uint32_t)(kTcBN * kTcBK * 2);
  P.Q = Q; P.nc = nc; P.Kp = Kp; P.nkb = (Kp + kTcBK - 1) / kTcBK;
  P.a_resident = Kp <= kTcResidentMaxK ? 1 : 0;
  const size_t budget = 227 * 1024 - 2048;   // opt-in shared memory of a block on sm_90, minus control block + alignment slack
  const size_t a_bytes = P.a_resident ? (size_t)P.nkb * 2 * P.tile_bytes : 0;
  const size_t st_bytes = (P.a_resident ? 2 : 4) * (size_t)P.tile_bytes;
  int nstages = (int)((budget - a_bytes) / st_bytes);
  if (nstages > kTcMaxStages) nstages = kTcMaxStages;
  if (nstages < 2) { set_error("tc_sweep: shared-memory plan failed"); return KGE_ENOTSUP; }
  P.nstages = nstages;
  P.ntiles = (int)((nc + kTcBN - 1) / kTcBN);
  const int qblocks = (int)((Q + kTcBM - 1) / kTcBM);
  // one CTA per SM: as many runs of tiles as fit in ONE wave over (directions x query blocks)
  int splits = sm_count() / (qblocks * ndirs);
  if (splits < 1) splits = 1;
  if (splits > P.ntiles) splits = P.ntiles;
  P.tiles_per_cta = (P.ntiles + splits - 1) / splits;
  splits = (P.ntiles + P.tiles_per_cta - 1) / P.tiles_per_cta;
  P.trace = g_tc_trace;
  // bf16 matrices [rows][Kp]; box = {64 columns (128 bytes), 128 rows}, 128-byte swizzle
  TcMaps TM;
  CUtensorMap* const maps[6] = {&TM.a0, &TM.a1, &TM.c0, &TM.c1, &TM.b0, &TM.b1};
  const size_t offs[6] = {L.a[dz[0]][0], L.a[dz[0]][1], L.a[dz[1]][0], L.a[dz[1]][1], L.b[0], L.b[1]};
  for (int k = 0; k < 6; ++k) {
    const int rc = make_tensor_map(maps[k], CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, C.ws + offs[k], (uint64_t)(k < 4 ? Q : nc),
                                   (uint64_t)Kp, (uint64_t)Kp * 2, kTcBK, kTcBN, CU_TENSOR_MAP_SWIZZLE_128B);
    if (rc) return rc;
  }
  const size_t smem = 2048 + a_bytes + (size_t)nstages * st_bytes;
  const int rc = smem_optin(tc_sweep_kernel, smem);
  if (rc) return rc;
  SweepProfile* sp = sweep_profile(dir);
  if (sp->armed) KGE_CUDA_OK(cudaEventRecord(sp->beg, st));
  tc_sweep_kernel<<<dim3((unsigned)splits, (unsigned)qblocks, (unsigned)ndirs), kTcThreads, smem, st>>>(P, TM);
  KGE_CHECK_LAUNCH("tc_sweep_kernel");
  if (sp->armed) { KGE_CUDA_OK(cudaEventRecord(sp->end, st)); sp->valid = true; sp->ndirs = ndirs; }
  return KGE_OK;
}

}  // namespace kge
