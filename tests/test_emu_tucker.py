"""CPU check of TuckER's CUDA kernels (pykg2vec_b200/csrc/kge_tucker.cuh and the tiled GEMM they launch) under the
host emulation (tests/emu/cuda_runtime.h: every CUDA thread of a block is a host thread), with the launch geometry of
the C-ABI launchers: core matrices, x_pre, its norm and x must equal the oracle (tests/oracle_tucker) bit for bit; the
backward's sums agree within fp32 accumulation error (the atomics' order is free).  A ThreadSanitizer build
(tests/emu/race_check_tucker.cpp) checks the shared-memory synchronisation of the two trunk kernels; its barrier-free
control build must be flagged.  The real kernels: tests/test_gpu_tucker.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import emu_build
import tucker_util as tu

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_tucker.cuh")
_p = tu._p


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.build("emu_tucker.cpp", "libemu_tucker.so", HEADERS))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _cores(emu, tabs, ids):
    p, keep = tu.tucker_struct(tabs)
    ids = tu._i64(ids)
    M = np.full((len(ids), p.d1 * p.d1), np.nan, dtype=np.float32)
    ws = np.zeros(2 * max(len(ids), 1) * p.d2, dtype=np.float32)
    emu.emu_tucker_cores(ctypes.byref(p), _p(ids), ctypes.c_int64(len(ids)), _p(M), _p(ws))
    return M


def _fwd(emu, tabs, M, e, slot, noise0=None, mask=None, noise2=None):
    p, keep = tu.tucker_struct(tabs)
    e, slot, noise0, noise2 = tu._i64(e), tu._i64(slot), tu._f32(noise0), tu._f32(noise2)
    ms, alive = tu.mask_struct(mask)
    Q = len(e)
    x, xpre = np.full((Q, p.d1), np.nan, np.float32), np.full((Q, p.d1), np.nan, np.float32)
    nrm = np.full(Q, np.nan, np.float32)
    emu.emu_tucker_trunk_fwd(ctypes.byref(p), _p(M), _p(e), _p(slot), ctypes.c_int64(Q), _p(noise0),
                             ctypes.byref(ms) if ms is not None else None, _p(noise2), _p(x), _p(xpre), _p(nrm))
    return x, xpre, nrm


def _bwd(emu, tabs, M, ids, e, slot, gx, xpre, nrm, noise0=None, mask=None, noise2=None):
    p, keep = tu.tucker_struct(tabs)
    ids, e, slot = tu._i64(ids), tu._i64(e), tu._i64(slot)
    noise0, noise2, gx = tu._f32(noise0), tu._f32(noise2), tu._f32(gx)
    ms, alive = tu.mask_struct(mask)
    gent, dM = np.zeros_like(keep[0]), np.zeros_like(M)
    grel, gW = np.zeros_like(keep[1]), np.zeros_like(keep[2])
    ws = np.zeros(2 * len(ids) * p.d2, dtype=np.float32)
    emu.emu_tucker_trunk_bwd(ctypes.byref(p), _p(M), _p(e), _p(slot), ctypes.c_int64(len(e)), _p(noise0),
                             ctypes.byref(ms) if ms is not None else None, _p(noise2), _p(gx), _p(xpre), _p(nrm),
                             _p(gent), _p(dM))
    emu.emu_tucker_cores_bwd(ctypes.byref(p), _p(ids), ctypes.c_int64(len(ids)), _p(dM), _p(grel), _p(gW), _p(ws))
    return gent, dM, grel, gW


@pytest.mark.parametrize("name", tu.CASES)
def test_emulated_forward_equals_oracle_bitwise_on_goldens(emu, name):
    g = tu.load(name)
    tabs = tu.tables(g)
    ids, slot = tu.slots(g["r"])
    M = _cores(emu, tabs, ids)
    assert _bits_equal(M, tu.oracle_cores(tabs, ids))
    nz = tu.noises(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        n0, n1, n2 = nz[tag] if nz else (None, None, None)
        mask = ("explicit", n1) if n1 is not None else None
        for got, want in zip(_fwd(emu, tabs, M, e, slot, n0, mask, n2), tu.oracle_trunk(tabs, M, e, slot, n0, mask, n2)):
            assert _bits_equal(got, want)


def _random_case(seed, N, R, d1, d2, Q, rels):
    rng = np.random.RandomState(seed)
    tabs = [rng.randn(N, d1).astype(np.float32), rng.randn(R, d2).astype(np.float32),
            (0.3 * rng.randn(d2, d1 * d1)).astype(np.float32)]
    e, r = rng.randint(N, size=Q), rng.choice(rels, size=Q)
    noise0 = ((rng.rand(Q, d1) > 0.3) / np.float32(0.7)).astype(np.float32)
    noise2 = ((rng.rand(Q, d1) > 0.5) / np.float32(0.5)).astype(np.float32)
    return rng, tabs, e, r, noise0, noise2


def test_cores_do_not_depend_on_the_other_relations_of_the_call(emu):
    """U = 70 spans two 64-row GEMM tiles with a ragged second one; a relation's matrix has the same bits alone, in
    any position and in any company; d1*d1 = 361 and d2 = 19 are not multiples of the tile sizes or of 4"""
    rng, tabs, *_ = _random_case(3, 7, 70, 19, 19, 1, [0])
    ids = rng.permutation(70)
    M = _cores(emu, tabs, ids)
    assert _bits_equal(M, tu.oracle_cores(tabs, ids))
    assert _bits_equal(_cores(emu, tabs, ids[5:6]), M[5:6])
    assert _bits_equal(_cores(emu, tabs, ids[[69, 5, 5]]), M[[69, 5, 5]])
    assert _cores(emu, tabs, ids[:0]).shape == (0, 361)


@pytest.mark.parametrize("mode", ["none", "explicit", "counter"])
def test_emulated_trunk_forward_and_backward(emu, mode):
    """queries sharing a relation and an entity, slot a permutation of the sorted order, odd widths"""
    N, R, d1, d2, Q, p = 9, 6, 21, 6, 7, 0.4
    rng, tabs, e, r, noise0, noise2 = _random_case(11, N, R, d1, d2, Q, [5, 0, 3])
    e[3] = e[0]
    ids = np.array([3, 5, 0])                                # not sorted: slot is a permutation of np.unique's
    slot = np.array([list(ids).index(v) for v in r])
    mask = {"none": None, "explicit": ("explicit", ((rng.rand(Q, d1, d1) > p) / np.float32(1 - p)).astype(np.float32)),
            "counter": ("counter", 2 ** 40 + 17, 2 ** 33 + 3, p)}[mode]
    M = _cores(emu, tabs, ids)
    x, xpre, nrm = _fwd(emu, tabs, M, e, slot, noise0, mask, noise2)
    for got, want in zip((x, xpre, nrm), tu.oracle_trunk(tabs, M, e, slot, noise0, mask, noise2)):
        assert _bits_equal(got, want)
    gx = rng.randn(Q, d1).astype(np.float32)
    got = _bwd(emu, tabs, M, ids, e, slot, gx, xpre, nrm, noise0, mask, noise2)
    gent, dM = tu.oracle_trunk_bwd(tabs, M, e, slot, gx, noise0, mask, noise2)
    grel, gW = tu.oracle_cores_bwd(tabs, ids, dM)
    # every output is a sum of at most Q * d1 * d1 fp32 products: n * 2^-24 relative to the largest magnitude is the
    # textbook bound for any summation order; the observed error is far below it
    for a, b in zip(got, (gent, dM, grel, gW)):
        assert np.abs(a - b).max() <= 64 * 2.0 ** -24 * np.abs(b).max()
    if mode == "counter":   # counter mode == explicit mode fed kge_tucker_mask1's values, bit for bit
        m1 = np.full((Q, d1, d1), np.nan, dtype=np.float32)
        emu.emu_tucker_mask1(ctypes.c_uint64(mask[1]), ctypes.c_uint64(mask[2]), ctypes.c_float(p), ctypes.c_int64(Q),
                             d1, _p(m1))
        assert _bits_equal(m1, tu.oracle_mask1(mask[1], mask[2], p, Q, d1))
        ex = ("explicit", m1)
        x2, xpre2, nrm2 = _fwd(emu, tabs, M, e, slot, noise0, ex, noise2)
        assert _bits_equal(x2, x) and _bits_equal(xpre2, xpre)
        # one query at a time (no two CTAs add to the same address): the backward is then deterministic too
        for q in range(Q):
            s = slice(q, q + 1)
            cm = ("counter", mask[1], mask[2] + q * d1 * d1, p)
            a = _bwd(emu, tabs, M, ids, e[s], slot[s], gx[s], xpre[s], nrm[s], noise0[s], cm, noise2[s])
            b = _bwd(emu, tabs, M, ids, e[s], slot[s], gx[s], xpre[s], nrm[s], noise0[s], ("explicit", m1[s]), noise2[s])
            assert all(_bits_equal(u, v) for u, v in zip(a[:2], b[:2]))


def test_full_width_rows(emu):
    """d1 = 256: every thread of the CTA owns a feature; d2 = 3"""
    rng, tabs, e, r, noise0, noise2 = _random_case(21, 4, 3, 256, 3, 2, [2, 1])
    ids, slot = tu.slots(r)
    M = _cores(emu, tabs, ids)
    assert _bits_equal(M, tu.oracle_cores(tabs, ids))
    for got, want in zip(_fwd(emu, tabs, M, e, slot), tu.oracle_trunk(tabs, M, e, slot)):
        assert _bits_equal(got, want)


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_tucker.cpp) ------------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_tucker.cpp", name, HEADERS + (os.path.join(emu_build.EMU, "emu_tucker.cpp"),),
                           extra=["-g", "-fsanitize=thread"] + extra, shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_tucker", [])
    probe = subprocess.run([exe, "probe"], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_tucker_trunk_kernels_are_race_free(race_checker):
    res = subprocess.run([race_checker], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_tucker -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_tucker_trunk(race_checker):
    """positive control: the same kernels with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_tucker_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
