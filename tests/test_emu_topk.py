"""CPU check (no GPU) of the batched top-k kernels of pykg2vec_b200/csrc/kge_topk.cuh under the host emulation of
tests/emu/ (emu_topk.cpp), with the launch geometry and shared-memory plan of the launchers in kge_topk.cu:

  * the row selection against a numpy lexsort on crafted rows (all-equal rows, NaN / +-0 / +-inf, n < k, filters
    that leave fewer than k candidates, duplicate filter entries, k = 1 and 256, tie groups straddling the
    threshold) at n = 1, 37, 14,541 (row kept in shared memory) and 123,182 (row streamed from global memory);
  * the kernel-model score producer bit for bit against the oracle's 1-vs-all sweep for every golden model, for
    tail, head and relation candidates;
  * a ThreadSanitizer build of the selection (race_check_topk.cpp), with a barrier-free control build that must
    be flagged.
The compiled kernels are checked on the H100 by tests/test_gpu_topk.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import golden_util as gu
import oracle

import emu_build
from topk_util import NAN_BITS, ref_topk

HEADERS = ("kge_common.cuh", "kge_models.cuh", "kge_topk.cuh")


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.build("emu_topk.cpp", "libemu_topk.so", HEADERS))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def run_select(emu, rows, k, descending=False, filters=None):
    """rows [R, n] fp32; filters: list of per-row id lists or None -> (ids [R,k], score bits [R,k], row in smem)"""
    rows = np.ascontiguousarray(rows, dtype=np.float32)
    R, n = rows.shape
    ptr = idx = None
    if filters is not None:
        ptr = np.zeros(R + 1, dtype=np.int64)
        ptr[1:] = np.cumsum([len(f) for f in filters])
        idx = np.concatenate([np.asarray(f, dtype=np.int64) for f in filters] + [np.zeros(0, np.int64)])
        if idx.size == 0:
            idx = np.zeros(1, dtype=np.int64)
    ids = np.zeros((R, k), dtype=np.int64)
    out = np.zeros((R, k), dtype=np.float32)
    rc = emu.emu_topk_select(_p(rows), ctypes.c_int64(R), ctypes.c_int64(n), ctypes.c_int(k), ctypes.c_int(descending),
                             _p(ptr), _p(idx), _p(ids), _p(out))
    assert rc in (0, 1)
    return ids, out.view(np.uint32), rc == 1


def check_rows(emu, rows, k, descending=False, filters=None):
    ids, bits, in_smem = run_select(emu, rows, k, descending, filters)
    for i, row in enumerate(np.asarray(rows, dtype=np.float32)):
        want_ids, want_bits = ref_topk(row, k, descending, filters[i] if filters is not None else None)
        assert np.array_equal(ids[i], want_ids), (i, ids[i][:12], want_ids[:12])
        assert np.array_equal(bits[i], want_bits), i
    return in_smem


def test_equal_scores_give_the_smallest_ids(emu):
    rows = np.full((2, 1000), 0.25, dtype=np.float32)
    rows[1] = -0.0
    for k in (1, 10, 256):
        ids, bits, _ = run_select(emu, rows, k)
        assert np.array_equal(ids, np.tile(np.arange(k), (2, 1)))
        check_rows(emu, rows, k)
    check_rows(emu, rows, 17, descending=True)


def test_nan_signed_zero_and_infinities(emu):
    rng = np.random.RandomState(1)
    specials = np.array([np.nan, -np.nan, 0.0, -0.0, np.inf, -np.inf, 1.5, -1.5], dtype=np.float32)
    rows = specials[rng.randint(len(specials), size=(3, 37))]
    rows[2, :5] = rng.standard_normal(5)
    for k in (1, 5, 20, 37, 256):
        for desc in (False, True):
            check_rows(emu, rows, k, descending=desc)


def test_fewer_candidates_than_k(emu):
    rng = np.random.RandomState(2)
    check_rows(emu, rng.standard_normal((2, 1)), 10)
    check_rows(emu, rng.standard_normal((2, 37)), 256)
    # a filter that leaves 5 of 300 candidates, with duplicate entries and ids outside the row
    keep = {3, 77, 150, 151, 299}
    filt = [i for i in range(300) if i not in keep] + [0, 0, 1, 2, 298, -1, 300, 10 ** 9]
    rows = rng.standard_normal((2, 300))
    ids, bits, _ = run_select(emu, rows, 10, filters=[filt, []])
    assert set(ids[0][:5]) == keep and np.all(ids[0][5:] == -1) and np.all(bits[0][5:] == NAN_BITS)
    check_rows(emu, rows, 10, filters=[filt, []])
    # everything filtered
    check_rows(emu, rows, 4, filters=[list(range(300)), list(range(300)) * 2])


@pytest.mark.parametrize("n", [1, 37, 14541, 123182])
def test_selection_matches_lexsort(emu, n):
    rng = np.random.RandomState(n)
    rows = [rng.standard_normal(n).astype(np.float32),
            rng.randint(0, 7, size=n).astype(np.float32) - 3.0,        # a tie group straddles the threshold
            (rng.standard_normal(n) * 1e-3).astype(np.float32)]
    if n >= 37:
        rows[2][rng.randint(n, size=n // 10 + 1)] = np.nan
        rows[2][rng.randint(n, size=n // 10 + 1)] = -0.0
    rows = np.stack(rows)
    filters = [rng.randint(n, size=min(n, 50)).tolist(), [], rng.randint(n, size=min(n, 3000)).tolist() * 2]
    in_smem = None
    for k in (1, 10, 256):
        in_smem = check_rows(emu, rows, k, filters=filters)
    check_rows(emu, rows[:2], 33, descending=True)
    assert in_smem == (n <= 14541)   # 123,182 candidates: the row is streamed from global memory


def test_threshold_tie_group_straddles_the_boundary(emu):
    # 30 strictly better candidates, then 200 ties at the threshold spread over the row: k = 100 takes 70 of them
    n = 2000
    row = np.full(n, 5.0, dtype=np.float32)
    rng = np.random.RandomState(3)
    better = rng.choice(n, 30, replace=False)
    row[better] = rng.standard_normal(30).astype(np.float32) - 10.0
    rest = np.setdiff1d(np.arange(n), better)
    ties = np.sort(rng.choice(rest, 200, replace=False))
    row[np.setdiff1d(rest, ties)] = 9.0
    row[ties] = 1.0
    ids, _, _ = run_select(emu, row[None], 100)
    assert np.array_equal(np.sort(ids[0][30:]), ties[:70])
    check_rows(emu, row[None], 100)
    check_rows(emu, row[None], 256, filters=[ties[:50].tolist()])


def test_chunking_bounds_the_workspace(emu):
    emu.emu_topk_chunk_rows.restype = ctypes.c_longlong
    rows = lambda Q, n: emu.emu_topk_chunk_rows(ctypes.c_longlong(Q), ctypes.c_longlong(n))
    assert rows(70000, 14541) == (64 << 20) // (4 * 14541)
    assert rows(70000, 37) == 65535
    assert rows(5, 37) == 5
    assert rows(3, 40_000_000) == 1


# ---- the kernel-model score producer vs the oracle ---------------------------------------------------------
def _widths(om):
    return [t.shape[-1] if t.ndim > 1 else 1 for t in om.tables]


@pytest.mark.parametrize("name", gu.case_names())
def test_store_producer_is_bit_exact(emu, name):
    g = gu.load(name)
    om = gu.oracle_model(g)
    if om.name == "rescal":            # Rescal.forward row-normalises its tables in place first
        for tab in om.tables:
            oracle.normalize_rows(tab)
    m = om.c_struct()
    Q = 3
    h, r, t = (np.ascontiguousarray(g[k][:Q], dtype=np.int64) for k in ("h", "r", "t"))
    vec = 4 if all(w % 4 == 0 for w in _widths(om)) and om.dim % 4 == 0 and om.name != "analogy" else 1
    for target in (0, 1, 2):
        n = om.num_rel if target == 2 else om.num_ent
        got = np.full((Q, n), np.nan, dtype=np.float32)
        rc = emu.emu_topk_store(ctypes.byref(m), ctypes.c_int(target), ctypes.c_int(vec),
                                _p(h) if target != 1 else None, _p(r) if target != 2 else None,
                                _p(t) if target != 0 else None, ctypes.c_int64(Q), _p(got))
        assert rc == 0
        for q in range(Q):
            if target == 0:
                want = oracle.sweep_scores(om, oracle.GROUP_TAIL, h[q], r[q], t[q])
            elif target == 1:
                want = oracle.sweep_scores(om, oracle.GROUP_HEAD, h[q], r[q], t[q])
            else:
                want = oracle.score_fwd(om, np.full(n, h[q]), np.arange(n), np.full(n, t[q]), oracle.GROUP_TAIL)
            assert np.array_equal(got[q].view(np.uint32), want.view(np.uint32)), (name, target, q)


# ---- ThreadSanitizer ---------------------------------------------------------------------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_topk.cpp", name, HEADERS, extra=["-g", "-fsanitize=thread"] + extra,
                           shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_topk", [])
    probe = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_selection_is_race_free(race_checker):
    res = subprocess.run([race_checker, "select"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, res.stderr[-3000:]


def test_race_detector_flags_a_missing_barrier(race_checker):
    """positive control: the selection with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_topk_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe, "select"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
