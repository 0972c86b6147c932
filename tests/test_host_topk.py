"""CPU tests (no GPU) of the batched top-k entry points: the C-ABI argument checks return before any launch, the
workspace bound, and the Evaluator's host-side refusals."""
import ctypes
import types

import numpy as np
import pytest

from pykg2vec_b200 import _lib
from pykg2vec_b200.evaluator import Evaluator

EINVAL, EWORKSPACE = -1, -4


def _model(N=100, R=5, d=8):
    m = _lib.KgeModel()
    m.model, m.dim, m.rel_dim, m.num_ent, m.num_rel = _lib.MODEL_IDS["transe"], d, d, N, R
    m.tables[0] = m.tables[1] = 16
    return m


def test_workspace_is_bounded_by_one_chunk():
    L = _lib.lib()
    i64, i32 = ctypes.c_int64, ctypes.c_int32
    assert L.kge_topk_workspace_bytes(i64(10), i64(1024), i32(10)) == 10 * 1024 * 4
    assert L.kge_topk_workspace_bytes(i64(70000), i64(14541), i32(10)) == (((64 << 20) // (4 * 14541)) * 14541 * 4 + 255) // 256 * 256
    assert L.kge_topk_workspace_bytes(i64(10 ** 6), i64(37), i32(1)) == (65535 * 37 * 4 + 255) // 256 * 256
    for bad in ((i64(-1), i64(10), i32(1)), (i64(1), i64(0), i32(1)), (i64(1), i64(10), i32(0)),
                (i64(1), i64(10), i32(257))):
        assert L.kge_topk_workspace_bytes(*bad) == 0


def test_argument_checks_stop_before_any_launch():
    L = _lib.lib()
    i64, i32 = ctypes.c_int64, ctypes.c_int32
    p = ctypes.c_void_p(16)
    m = _model()
    before = L.kge_launch_count()
    big = i64(1 << 30)

    def topk(target=0, qh=p, qr=p, qt=p, Q=3, k=10, ids=p, sc=p, ws=p, wsb=big, fptr=None, fidx=None, fnnz=0):
        return L.kge_topk_1vsall(ctypes.byref(m), i32(target), qh, qr, qt, i64(Q), i32(k), fptr, fidx, i64(fnnz),
                                 ids, sc, ws, wsb, None)

    def ptopk(Q=3, N=100, width=8, k=10, ids=p, sc=p, ws=p, wsb=big):
        return L.kge_proj_topk(p, p, None, i64(Q), i64(N), i32(width), i32(k), None, None, i64(0), ids, sc, ws, wsb,
                               None)

    for k in (0, 257, -3):
        assert topk(k=k) == EINVAL and ptopk(k=k) == EINVAL
    for target in (-1, 3):
        assert topk(target=target) == EINVAL
    assert topk(Q=-1) == EINVAL and ptopk(Q=-1) == EINVAL
    assert topk(ids=None) == EINVAL and topk(sc=None) == EINVAL and topk(ws=None) == EINVAL
    assert ptopk(ids=None) == EINVAL and ptopk(sc=None) == EINVAL and ptopk(width=0) == EINVAL
    assert topk(qh=None) == EINVAL and topk(target=1, qt=None) == EINVAL and topk(target=2, qh=None) == EINVAL
    assert topk(fnnz=5) == EINVAL                          # a filter without its arrays
    assert topk(wsb=i64(3 * 100 * 4 - 1)) == EWORKSPACE
    assert topk(target=2, wsb=i64(3 * 5 * 4 - 1)) == EWORKSPACE
    assert ptopk(wsb=i64(3 * 100 * 4 - 1)) == EWORKSPACE
    assert topk(Q=0, ids=None, sc=None, ws=None) == 0 and ptopk(Q=0, ids=None, sc=None, ws=None) == 0
    assert L.kge_launch_count() == before


def test_evaluator_refusals_need_no_device():
    ev = Evaluator.__new__(Evaluator)
    ev.model = types.SimpleNamespace(proj_query=lambda *a, **k: None)
    ev.config = types.SimpleNamespace(device="cpu", tot_entity=50, tot_relation=4)
    with pytest.raises(_lib.KgeNotSupported):
        ev.predict_rels([0], [1])
    ev.model = types.SimpleNamespace()
    for call in (lambda: ev.predict_tails([0, 50], [0, 1]), lambda: ev.predict_tails([0], [4]),
                 lambda: ev.predict_heads([0], [-1]), lambda: ev.predict_rels([0], [50]),
                 lambda: ev.predict_tails([0, 1], [0]), lambda: ev.predict_tails([0], [0], k=0),
                 lambda: ev.predict_heads([0], [0], k=257)):
        with pytest.raises(ValueError):
            call()
    assert np.asarray(ev._topk_ids([3, 4], 5, "h")).dtype == np.int64
