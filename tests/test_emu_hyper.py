"""CPU check of HypER's inference-trunk CUDA kernels (pykg2vec_b200/csrc/kge_hyper.cuh) under the host
emulation (tests/emu/cuda_runtime.h: every CUDA thread of a block is a host thread), through the same
workspace layout and launch plans as the C-ABI launcher: the filter table (tiled GEMM), the features
(gather + bn0 + per-query conv + bn1), the sliced Linear GEMM and the bn2 + ReLU combine must equal the
oracle bit for bit — on the reference's own parameters and at the FB15k-237 width (de = dr = 200).
A ThreadSanitizer build of the same kernels (tests/emu/race_check_hyper.cpp) checks their shared-memory
synchronisation; its barrier-free control build must be flagged.
The real kernels are checked on the GPU by tests/test_gpu_hyper.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import emu_build
import hyper_util as hu

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_conve.cuh", "kge_hyper.cuh")


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(emu_build.build("emu_hyper.cpp", "libemu_hyper.so", HEADERS))
    L.emu_hyper_workspace_floats.restype = ctypes.c_int64
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(emu, st, e, r):
    """-> (x, filter table, features) of the emulated kernels"""
    p, keep = hu.hyper_struct(st)
    e, r = np.ascontiguousarray(e, dtype=np.int64), np.ascontiguousarray(r, dtype=np.int64)
    Q, de, R = len(e), p.ent_hidden_size, p.num_rel
    ws = np.full(emu.emu_hyper_workspace_floats(ctypes.c_int64(R), ctypes.c_int64(Q), ctypes.c_int32(de)), np.nan,
                 dtype=np.float32)
    fo, go = ctypes.c_int64(), ctypes.c_int64()
    emu.emu_hyper_layout(ctypes.c_int64(R), ctypes.c_int64(Q), ctypes.c_int32(de), ctypes.byref(fo), ctypes.byref(go))
    x = np.full((Q, de), np.nan, dtype=np.float32)
    emu.emu_hyper_trunk_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), _p(x), _p(ws))
    F = 32 * (de - 8)
    return x, ws[fo.value:fo.value + R * 288].reshape(R, 288), ws[go.value:go.value + Q * F].reshape(Q, F)


def _bits_equal(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", hu.CASES)
def test_emulated_trunk_bit_exact_on_reference_parameters(emu, name):
    g = hu.load(name)
    st = hu.state(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        x, filt, feat = _run(emu, st, e, g["r"])
        wx, wfilt, wfeat = hu.oracle_trunk_fwd(st, e, g["r"], intermediates=True)
        assert _bits_equal(filt, wfilt), "filter GEMM"
        assert _bits_equal(feat, wfeat), "feature kernel"
        assert _bits_equal(x, wx), "Linear + combine"
        assert np.abs(x - g["x_" + tag]).max() <= 1e-5


def test_emulated_trunk_bit_exact_at_fb15k237_width(emu):
    """de = dr = 200 (hyperparams/HypER.yaml): 12 Linear slices of 512 features, Q = 77 (two row tiles)"""
    N, R, de, dr, Q = 300, 237, 200, 200, 77
    st = hu.random_state(N, R, de, dr, seed=77)
    rng = np.random.RandomState(5)
    e, r = rng.randint(N, size=Q), rng.randint(R, size=Q)
    e[:3], r[:3] = 0, 0
    x, filt, feat = _run(emu, st, e, r)
    wx, wfilt, wfeat = hu.oracle_trunk_fwd(st, e, r, intermediates=True)
    assert _bits_equal(filt, wfilt) and _bits_equal(feat, wfeat) and _bits_equal(x, wx)
    assert (x > 0).any() and (x == 0).any()       # the ReLU is live on both sides


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_hyper.cpp) ---------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_hyper.cpp", name, HEADERS, extra=["-g", "-fsanitize=thread"] + extra,
                           shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_hyper", [])
    probe = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_hyper_trunk_kernels_are_race_free(race_checker):
    res = subprocess.run([race_checker, "trunk"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_hyper trunk -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_hyper_trunk(race_checker):
    """positive control: the same kernels with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_hyper_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe, "trunk"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
