"""-m gpu test of the tensor-core sweep's timeline aid (kge_debug_set_tc_trace, read by profiles/tc_trace.py): at the
bench's evaluation shape every event of CTA (0,0,0) leaves exactly one stamp, in its own role's slots and in time
order, and a traced call counts exactly what an untraced one does."""
import ctypes

import numpy as np
import pytest
import torch

import golden_util as gu

pytestmark = pytest.mark.gpu


def test_timeline_has_one_stamp_per_event_in_its_own_slots():
    from pykg2vec_b200 import _lib
    spec = gu.BASELINE_SHAPES["cfg2_transe_fb15k237"]
    desc = _lib.ModelDesc(spec["model"], [torch.from_numpy(t).cuda() for t in gu.baseline_tables(spec)], spec["d"],
                          l1_flag=spec["l1"], margin=spec["margin"])
    rng = np.random.RandomState(1)
    Q = 512
    q = [torch.from_numpy(rng.randint(n, size=Q)).cuda() for n in (spec["N"], spec["R"], spec["N"])]
    want = _lib.rank_1vsall(desc, *q).cpu().numpy()

    buf = torch.zeros(3 * 64 + 2048, dtype=torch.int64, device="cuda")
    _lib.lib().kge_debug_set_tc_trace(ctypes.c_void_p(buf.data_ptr()))
    try:
        got = _lib.rank_1vsall(desc, *q).cpu().numpy()
    finally:
        _lib.lib().kge_debug_set_tc_trace(ctypes.c_void_p(0))
    np.testing.assert_array_equal(got, want)

    # the launch's geometry (tc_sweep): Kp = 208 -> 4 k-blocks per tile; runs of tiles sized to one wave of CTAs
    # over (2 directions x 4 query blocks)
    nkb = 4
    ntiles = (spec["N"] + 127) // 128
    splits = min(max(torch.cuda.get_device_properties(0).multi_processor_count // 8, 1), ntiles)
    ntl = (ntiles + splits - 1) // splits
    assert 1 + ntl * nkb <= 61, "the shape leaves more events than the timeline has slots"
    t = buf.cpu().numpy()[:192].reshape(3, 64)
    nz = lambda row: np.flatnonzero(row[:62])
    # producer: start + one stamp per k-block issued; consumer (warp 4): start + one per full-barrier wait
    assert list(nz(t[0])) == list(range(1 + ntl * nkb))
    assert list(nz(t[1])) == list(range(1 + ntl * nkb))
    # epilogue begin / end per tile in slots 1 .. 2 ntl; slot 63 = kernel entry, 62 = exit
    assert list(nz(t[2])) == list(range(1, 1 + 2 * ntl))
    for r, slots in ((0, nz(t[0])), (1, nz(t[1])), (2, nz(t[2]))):
        assert np.all(np.diff(t[r, slots]) >= 0), r
    entry, leave = t[2, 63], t[2, 62]
    assert entry <= t[0, 0] and entry <= t[1, 0] and t[2, 2 * ntl] <= leave
    assert 0 <= t[1, 63] <= leave - entry   # cycles inside full-barrier waits
