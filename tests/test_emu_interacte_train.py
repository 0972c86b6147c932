"""CPU check of InteractE's training-mode trunk kernels (pykg2vec_b200/csrc/kge_interacte_train.cuh, the
kge_conve_train.cuh kernels and the tiled GEMM they launch) under the host emulation (tests/emu/cuda_runtime.h: every
CUDA thread of a block is a host thread), with the launch sequence of kge_interacte_train_fwd / _bwd: x and the running
statistics must equal the oracle (tests/oracle_interacte_train) bit for bit, the tail and head forwards as one call
over two groups; the backward agrees with the oracle's fp64 backward within the fp32 summation bound.  A
ThreadSanitizer build (tests/emu/race_check_interacte_train.cpp) checks the shared-memory synchronisation of the
CTA-per-query kernels; its barrier-free control build must be flagged.  The real kernels:
tests/test_gpu_interacte_train.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import emu_build
import interacte_train_util as itu

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_conve.cuh", "kge_conve_train.cuh", "kge_hyper.cuh",
           "kge_interacte.cuh", "kge_interacte_train.cuh")
_p = itu._p


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.build("emu_interacte_train.cpp", "libemu_interacte_train.so", HEADERS))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def emu_fwd(emu, sd, e, r, B, n0=None, n1=None, n2=None, running=None):
    """the emulated forward -> (x, workspace); `running` (a dict) receives the updated running statistics"""
    p, keep = itu.model_struct(sd)
    e, r, n0, n1, n2 = itu._i64(e), itu._i64(r), itu._f32(n0), itu._f32(n1), itu._f32(n2)
    Q = len(e)
    emu.emu_interacte_train_workspace_floats.restype = ctypes.c_int64
    ws = np.zeros(emu.emu_interacte_train_workspace_floats(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)),
                  np.float32)
    x = np.full((Q, p.reshape_height * p.reshape_width), np.nan, np.float32)
    emu.emu_interacte_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), ctypes.c_int64(B), _p(n0), _p(n1),
                                _p(n2), _p(x), _p(ws))
    if running is not None:
        running.update({key: keep[key] for key in itu.RUNNING})
    return x, ws


def emu_bwd(emu, sd, e, r, B, gx, x, ws, n0=None, n1=None, n2=None):
    p, keep = itu.model_struct(sd, running=False)
    e, r, n0, n1, n2 = itu._i64(e), itu._i64(r), itu._f32(n0), itu._f32(n1), itu._f32(n2)
    grads = [np.zeros(np.shape(sd[key]), np.float32) for key in itu.PARAMS]
    arr = (ctypes.c_void_p * len(grads))(*[g.ctypes.data for g in grads])
    emu.emu_interacte_train_bwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B), _p(n0),
                                _p(n1), _p(n2), _p(itu._f32(gx)), _p(itu._f32(x)), arr, _p(ws))
    return grads


def _both_directions(g):
    """the tail and head rows of a golden case as one call of two groups, with the reference's noise"""
    B = len(g["h"])
    e, r = np.concatenate([g["h"], g["t"]]), np.concatenate([g["r"], g["r"]])
    nt, nh = itu.noises(g, "tail"), itu.noises(g, "head")
    nz = [None if a is None else np.concatenate([a, b]) for a, b in zip(nt, nh)]
    return e, r, B, nz


@pytest.mark.parametrize("name", itu.CASES)
def test_emulated_forward_equals_oracle_bitwise_on_goldens(emu, name):
    g = itu.load(name)
    sd = itu.state(g)
    e, r, B, nz = _both_directions(g)
    run_e, run_o = {}, {}
    x, _ = emu_fwd(emu, sd, e, r, B, *nz, running=run_e)
    want = itu.oracle_fwd(sd, e, r, B, *nz, running=run_o)
    assert _bits_equal(x, want)
    for key in itu.RUNNING:
        assert _bits_equal(run_e[key], run_o[key]), key
        assert np.abs(run_e[key] - g["sd_after_" + key]).max() < 1e-5, key   # = the reference's two forwards


@pytest.mark.parametrize("name", itu.CASES)
def test_emulated_backward_within_the_fp32_bound(emu, name):
    g = itu.load(name)
    sd = itu.state(g)
    e, r, B, nz = _both_directions(g)
    x, ws = emu_fwd(emu, sd, e, r, B, *nz)
    gx = np.random.RandomState(5).randn(len(e), x.shape[1]).astype(np.float32)
    got = emu_bwd(emu, sd, e, r, B, gx, x, ws, *nz)
    want, _ = itu.oracle_bwd64(sd, e, r, B, gx, *nz)
    scale = max(np.abs(w).max() for w in want)
    # each output is a sum of at most B * P * F * 2k fp32 terms per group; the fp32 arithmetic of the statistics and
    # of every BatchNorm backward adds relative rounding of order 2^-24 per step: 1e-4 of the output's largest
    # magnitude bounds them; bn0's affine parameters and fc.bias (true gradient ~0 in front of a training-mode
    # BatchNorm with dropouts 0) are held to the step's scale
    for key, a, b in zip(itu.PARAMS, got, want):
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max() + 1e-6 * scale, key


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_interacte_train.cpp) ---------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_interacte_train.cpp", name,
                           HEADERS + (os.path.join(emu_build.EMU, "emu_interacte_train.cpp"),),
                           extra=["-g", "-fsanitize=thread"] + extra, shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_interacte_train", [])
    probe = subprocess.run([exe, "probe"], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_interacte_train_kernels_are_race_free(race_checker):
    res = subprocess.run([race_checker], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_interacte_train -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_interacte_train_kernels(race_checker):
    """positive control: the same kernels with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_interacte_train_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
