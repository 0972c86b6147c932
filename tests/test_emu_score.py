"""CPU check (no GPU) of the per-model score functions in pykg2vec_b200/csrc/kge_models.cuh — the
device math behind kge_score_fwd and the gather sweep — run under the host emulation of
tests/emu/ with the thread mapping of score_fwd_kernel, against the oracle, BIT FOR BIT, on the
tables of every golden case (both groupings).  A regression net for the model math that needs no
GPU; the compiled kernels themselves are checked on the GPU by tests/test_gpu_score_rank.py."""
import ctypes

import numpy as np
import pytest

import golden_util as gu
import oracle

import emu_build

CASES = [n for n in gu.case_names()]


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.models_lib())


def _widths(om):
    return [t.shape[-1] if t.ndim > 1 else 1 for t in om.tables]


@pytest.mark.parametrize("name", CASES)
def test_emulated_score_functions_are_bit_exact(emu, name):
    g = gu.load(name)
    om = gu.oracle_model(g)
    m = om.c_struct()
    n = min(40, len(g["h"]))           # 2 CTAs, the second one partly idle
    h, r, t = (np.ascontiguousarray(g[k][:n], dtype=np.int64) for k in ("h", "r", "t"))
    if om.name == "rescal":            # Rescal.forward row-normalises its tables in place first
        for tab in om.tables:
            oracle.normalize_rows(tab)
    # 16-byte row loads are legal when every row width is a multiple of 4 floats (numpy buffers are
    # 16-byte aligned); the scalar path is always legal and must give the same bits
    vecs = [1] + ([4] if all(w % 4 == 0 for w in _widths(om)) and om.dim % 4 == 0 else [])
    if om.name in ("analogy",) and (om.dim // 2) % 4:
        vecs = [1]
    for grouping in (oracle.GROUP_TAIL, oracle.GROUP_HEAD):
        want = oracle.score_fwd(om, h, r, t, grouping)
        for vec in vecs:
            got = np.full(n, np.nan, dtype=np.float32)
            rc = emu.emu_score_fwd(ctypes.byref(m), ctypes.c_int(grouping), ctypes.c_int(vec),
                                   h.ctypes.data_as(ctypes.c_void_p), r.ctypes.data_as(ctypes.c_void_p),
                                   t.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(n),
                                   got.ctypes.data_as(ctypes.c_void_p))
            assert rc == 0
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (name, grouping, vec)


# ---- backward: grad_group<MODEL, VEC> of kge_grads.cuh vs the reference's own autograd -------------
GRAD_TOL = 2e-4   # relative to the largest |gradient| of the table (as tests/test_gpu_train.py)


@pytest.fixture(scope="module")
def emu_bwd(emu):
    return emu


@pytest.mark.parametrize("name", [n for n in CASES if "pretrained" not in n])
def test_emulated_gradients_match_reference_autograd(emu_bwd, name):
    g = gu.load(name)
    om = gu.oracle_model(g)
    m = om.c_struct()
    h, r, t = (np.ascontiguousarray(g[k], dtype=np.int64) for k in ("h", "r", "t"))
    up = np.ascontiguousarray(g["upstream"], dtype=np.float32)
    grads = [np.zeros_like(tab) for tab in om.tables]
    arr = (ctypes.c_void_p * 16)()
    for k, a in enumerate(grads):
        arr[k] = a.ctypes.data
    vec = 4 if (all(w % 4 == 0 for w in _widths(om)) and om.dim % 4 == 0 and not (om.name == "analogy" and (om.dim // 2) % 4)) else 1
    rc = emu_bwd.emu_score_bwd(ctypes.byref(m), ctypes.c_int(vec), ctypes.c_int(len(grads)),
                               h.ctypes.data_as(ctypes.c_void_p), r.ctypes.data_as(ctypes.c_void_p),
                               t.ctypes.data_as(ctypes.c_void_p), ctypes.c_int64(len(h)),
                               up.ctypes.data_as(ctypes.c_void_p), arr)
    assert rc == 0
    for k, got in enumerate(grads):
        if "grad%d" % k not in g:      # ConvKB: no reference gradient for the collapsed tables
            continue
        want = np.asarray(g["grad%d" % k], dtype=np.float64).reshape(got.shape)
        scale = max(np.abs(want).max(), 1e-12)
        err = np.abs(got.astype(np.float64) - want).max() / scale
        assert err < GRAD_TOL, "%s table %d: rel err %.3g" % (name, k, err)
