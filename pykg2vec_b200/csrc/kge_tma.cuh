// kge_tma.cuh — Hopper async-copy helpers shared by the two 1-vs-all sweeps (kge_rank_tiled.cu,
// kge_rank_tc.cu): mbarriers, 2-D TMA tile loads and the tensor maps that describe them.
#pragma once
#include <cuda.h>  // CUtensorMap (driver types only; the encoder is fetched through the runtime)

#include "kge_common.cuh"

namespace kge {

// ---- device side ---------------------------------------------------------------------------------
KGE_DEV uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
KGE_DEV void mbar_init(uint64_t* bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
KGE_DEV void mbar_arrive_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
KGE_DEV void mbar_arrive(uint64_t* bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
// Bounded wait: a protocol bug must end in a trap (a loud launch failure), never in a hung GPU.
KGE_DEV void mbar_wait(uint64_t* bar, uint32_t parity) {
  const uint32_t addr = smem_u32(bar);
  const long long t0 = clock64();
  for (;;) {
    uint32_t ok;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(ok) : "r"(addr), "r"(parity) : "memory");
    if (ok) return;
    if (clock64() - t0 > 4000000000LL) __trap();   // ~2 s at 1.98 GHz
  }
}
// 2-D tensor-map tile load (TMA): box at (col, row) of the map's matrix into shared memory at dst_smem;
// out-of-bounds elements are zero-filled and still counted in the transaction bytes.
KGE_DEV void tma_load_2d(uint32_t dst_smem, const CUtensorMap* tm, int col, int row, uint64_t* bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
      ::"r"(dst_smem), "l"(reinterpret_cast<uint64_t>(tm)), "r"(col), "r"(row), "r"(smem_u32(bar))
      : "memory");
}

// ---- host side -----------------------------------------------------------------------------------
// Row-major matrix [rows][cols] of `dtype` with a row pitch of `pitch_bytes`; box {box_cols, box_rows};
// out-of-range elements read as zeros.  cuTensorMapEncodeTiled is reached through the runtime's
// driver-entry-point lookup (no -lcuda link).
int make_tensor_map(CUtensorMap* tm, CUtensorMapDataType dtype, const void* base, uint64_t rows, uint64_t cols,
                    uint64_t pitch_bytes, uint32_t box_cols, uint32_t box_rows, CUtensorMapSwizzle swizzle);

}  // namespace kge
