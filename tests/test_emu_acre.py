"""CPU check of AcrE's inference-trunk CUDA kernels (pykg2vec_b200/csrc/kge_acre.cuh) under the host emulation
(tests/emu/cuda_runtime.h: every CUDA thread of a block is a host thread), through the same workspace layout and
launch plans as the C-ABI launcher: the serial features (gather + bn0 + three chained atrous convs + residual +
bn1 + ReLU), the parallel way's gate input, W_gate_e GEMM and bn1 + ReLU, the sliced Linear GEMM and the bn2 +
ReLU combine must equal the oracle bit for bit — on the reference's own parameters and at in_channels 32 with
Q = 33, both ways.  A ThreadSanitizer build of the serial kernel (tests/emu/race_check_acre.cpp) checks its
shared-memory synchronisation; its barrier-free control build must be flagged.
The real kernels are checked on the GPU by tests/test_gpu_acre.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import acre_util as au
import emu_build

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_conve.cuh", "kge_hyper.cuh", "kge_acre.cuh")


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(emu_build.build("emu_acre.cpp", "libemu_acre.so", HEADERS))
    L.emu_acre_workspace_floats.restype = ctypes.c_int64
    L.emu_acre_smem_bytes.restype = ctypes.c_int64
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(emu, st, e, r):
    """-> (x, features, gate input or None) of the emulated kernels"""
    p, keep = au.acre_struct(st)
    e, r = np.ascontiguousarray(e, dtype=np.int64), np.ascontiguousarray(r, dtype=np.int64)
    Q, C = len(e), p.in_channels
    ws = np.full(emu.emu_acre_workspace_floats(ctypes.byref(p), ctypes.c_int64(Q)), np.nan, dtype=np.float32)
    x = np.full((Q, 200), np.nan, dtype=np.float32)
    assert emu.emu_acre_trunk_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), _p(x), _p(ws)) == 0
    off = np.zeros(3, dtype=np.int64)
    emu.emu_acre_layout(ctypes.byref(p), ctypes.c_int64(Q), _p(off))
    feat = ws[off[1]:off[1] + Q * C * 400].reshape(Q, C * 400)
    gate = ws[off[0]:off[0] + Q * C * 1600].reshape(Q * C, 1600) if p.way == 1 else None
    return x, feat, gate


def _bits_equal(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", au.CASES)
def test_emulated_trunk_bit_exact_on_reference_parameters(emu, name):
    g = au.load(name)
    st = au.state(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        x, feat, gate = _run(emu, st, e, g["r"])
        wx, wfeat, wgate = au.oracle_trunk_fwd(st, e, g["r"], intermediates=True)
        if gate is not None:
            assert _bits_equal(gate, wgate), "gate-input kernel"
        assert _bits_equal(feat, wfeat), "features"
        assert _bits_equal(x, wx), "Linear + combine"
        assert np.abs(x - g["x_" + tag]).max() <= 1e-5


@pytest.mark.parametrize("way", ["serial", "parallel"])
def test_emulated_trunk_bit_exact_at_32_channels(emu, way):
    """in_channels 32, rates 1 / 2 / 2 (the yaml's) with conv bias, Q = 33 (an id 0 in both columns)"""
    N, R, Q = 300, 237, 33
    st = au.random_state(N, R, (way, 32, (1, 2, 2), True), seed=41)
    rng = np.random.RandomState(5)
    e, r = rng.randint(N, size=Q), rng.randint(2 * R, size=Q)
    e[:3], r[:3] = 0, 0
    x, feat, gate = _run(emu, st, e, r)
    wx, wfeat, wgate = au.oracle_trunk_fwd(st, e, r, intermediates=True)
    if gate is not None:
        assert _bits_equal(gate, wgate)
    assert _bits_equal(feat, wfeat) and _bits_equal(x, wx)
    assert (x > 0).any() and (x == 0).any() and (feat == 0).any()       # both ReLUs are live


def test_emulated_trunk_with_rates_beyond_the_image(emu):
    """rates >= 20 leave only the centre tap inside the image (serial, 9 channels, no conv bias)"""
    N, R, Q = 40, 5, 3
    st = au.random_state(N, R, ("serial", 9, (20, 1, 37), False), seed=8)
    e, r = np.array([0, 7, 39]), np.array([0, 9, 3])
    x, feat, _ = _run(emu, st, e, r)
    wx, wfeat, _ = au.oracle_trunk_fwd(st, e, r, intermediates=True)
    assert _bits_equal(feat, wfeat) and _bits_equal(x, wx)


def test_shared_memory_bound():
    """the serial kernel's layout fits 227 KB up to 46 channels (the bound stated in kge_acre.cuh); 141 KB at the
    yaml's 32"""
    def serial_bytes(C):
        cp = (C + 7) // 8 * 8
        return 4 * (400 + 800 * C + 9 * C * cp + 3 * cp)
    assert serial_bytes(32) == 141248
    assert serial_bytes(46) <= 227 * 1024 < serial_bytes(47)


def test_emulated_smem_sizes_match_the_stated_layout(emu):
    for C in (1, 9, 32, 46):
        st = au.random_state(4, 2, ("serial", C, (1, 2, 2), True), seed=1)
        p, keep = au.acre_struct(st)
        cp = (C + 7) // 8 * 8
        assert emu.emu_acre_smem_bytes(ctypes.byref(p)) == 4 * (400 + 800 * C + 9 * C * cp + 3 * cp)
        p.way = 1
        assert emu.emu_acre_smem_bytes(ctypes.byref(p)) == 4 * (400 + 30 * C)


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_acre.cpp) ---------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_acre.cpp", name, HEADERS, extra=["-g", "-fsanitize=thread"] + extra,
                           shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_acre", [])
    probe = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_acre_serial_kernel_is_race_free(race_checker):
    res = subprocess.run([race_checker, "serial"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_acre serial -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_acre_kernel(race_checker):
    """positive control: the same kernel with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_acre_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe, "serial"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
