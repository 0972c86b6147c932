"""measurement aid: timeline of one tc_sweep_kernel CTA (clock64 stamps) at the bench shape"""
import ctypes, json, sys, os
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import golden_util as gu
from pykg2vec_b200 import _lib
spec = gu.BASELINE_SHAPES[sys.argv[1] if len(sys.argv) > 1 else "cfg2_transe_fb15k237"]
tables = gu.baseline_tables(spec)
phase = float(np.float32(np.pi / ((spec["margin"] + 2.0) / spec["d"]))) if spec["model"] == "rotate" else 0.0
desc = _lib.ModelDesc(spec["model"], [torch.from_numpy(t).cuda() for t in tables], spec["d"], l1_flag=spec["l1"], margin=spec["margin"], phase_scale=phase)
rng = np.random.RandomState(0)
Q = 512
q = [torch.from_numpy(rng.randint(n, size=Q)).cuda() for n in (spec["N"], spec["R"], spec["N"])]
FL = 0 if os.environ.get("TC_TRACE_BOTH") else _lib.RANK_TAIL_ONLY   # TC_TRACE_BOTH=1: the product launch (both directions)
buf = torch.zeros(3 * 64 + 2048, dtype=torch.int64, device="cuda")
flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
for rep in range(3):
    _lib.rank_1vsall(desc, *q, flags=FL)
torch.cuda.synchronize()
buf.zero_()
# untraced timing first (mean of 5, L2 flushed)
times = []
for rep in range(5):
    flush.zero_(); torch.cuda.synchronize()
    _lib.rank_1vsall(desc, *q, flags=FL | _lib.RANK_PROFILE)
    torch.cuda.synchronize()
    times.append(_lib.rank_last_sweep_ms(0))
_lib.lib().kge_debug_set_tc_trace(ctypes.c_void_p(buf.data_ptr()))
flush.zero_(); torch.cuda.synchronize()
_lib.rank_1vsall(desc, *q, flags=FL | _lib.RANK_PROFILE)
torch.cuda.synchronize()
ms = _lib.rank_last_sweep_ms(0)
_lib.lib().kge_debug_set_tc_trace(ctypes.c_void_p(0))
raw = buf.cpu().numpy()
t = raw[:192].reshape(3, 64)
spans = raw[192:].reshape(1024, 2)
spans = spans[spans[:, 0] != 0]
t0 = t[2, 63]
out = {"directions": _lib.rank_last_sweep_directions(), "kernel_ms_untraced": times, "kernel_ms_traced": ms}
# role 0: the TMA producer's start, then one stamp per k-block issued (after its empty-barrier wait);
# 1: consumer warpgroup start (warp 4), then one stamp per k-block after its full-barrier wait;
# 2: epilogue begin / end per tile
for r, name in enumerate(("producer", "consumer", "epilogue")):
    out[name] = [int(x - t0) for x in t[r, :62] if x != 0]
prod, full, epi = out["producer"][1:], out["consumer"][1:], out["epilogue"]
ntile = len(epi) // 2
nkb = len(full) // ntile if ntile else 0
# per tile: first k-block's operands in hand -> last MMA retired (compare with the tensor time of a tile)
out["tile_mma_span_cycles"] = [epi[2 * i] - full[nkb * i] for i in range(ntile)] if nkb else []
# per k-block: the producer's TMA issue -> the consumer past the full barrier (about one TMA round trip when
# the consumers wait for operands, longer when the operands wait in the ring for the MMAs)
out["ready_lag_cycles"] = [f - p for f, p in zip(full, prod)]
out["starved_cycles"] = int(t[1, 63])   # warp 4's cycles inside full-barrier waits, summed
if len(spans):
    s0 = spans[:, 0].min()
    out["ctas"] = int(len(spans))
    out["cta_start_ns_minmax"] = [0, int(spans[:, 0].max() - s0)]
    out["cta_end_ns_minmax"] = [int(spans[:, 1].min() - s0), int(spans[:, 1].max() - s0)]
    out["cta0_ns"] = int(spans[0, 1] - spans[0, 0]) if raw[192] else None
    out["cta0_cycles"] = int(t[2, 62] - t0)
    out["cta_duration_ns_percentiles_0_50_100"] = [int(x) for x in np.percentile(spans[:, 1] - spans[:, 0], [0, 50, 100])]
print(json.dumps(out))
