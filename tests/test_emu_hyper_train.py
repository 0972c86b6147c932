"""CPU check of HypER's training-mode trunk kernels (pykg2vec_b200/csrc/kge_hyper_train.cuh, the kge_conve_train.cuh
kernels and the tiled GEMM they launch) under the host emulation (tests/emu/cuda_runtime.h: every CUDA thread of a
block is a host thread), with the launch sequence of kge_hyper_train_fwd / _bwd: x and the running statistics must
equal the oracle (tests/oracle_hyper_train) bit for bit, the tail and head forwards as one call over two groups; the
backward agrees with the oracle's fp64 backward within the fp32 summation bound.  A ThreadSanitizer build
(tests/emu/race_check_hyper_train.cpp) checks the shared-memory synchronisation of the CTA-per-query kernels; its
barrier-free control build must be flagged.  The real kernels: tests/test_gpu_hyper_train.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import emu_build
import hyper_train_util as hu

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_conve.cuh", "kge_conve_train.cuh", "kge_hyper.cuh", "kge_tucker.cuh",
           "kge_hyper_train.cuh")
_p = hu._p


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.build("emu_hyper_train.cpp", "libemu_hyper_train.so", HEADERS))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def emu_fwd(emu, sd, e, r, B, n0=None, n1=None, n2=None, running=None):
    """the emulated forward -> (x, workspace); `running` (a dict) receives the updated running statistics"""
    p, keep = hu.model_struct(sd)
    e, r, n0, n1, n2 = hu._i64(e), hu._i64(r), hu._f32(n0), hu._f32(n1), hu._f32(n2)
    Q = len(e)
    emu.emu_hyper_train_workspace_floats.restype = ctypes.c_int64
    ws = np.zeros(emu.emu_hyper_train_workspace_floats(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)),
                  np.float32)
    x = np.full((Q, p.ent_hidden_size), np.nan, np.float32)
    emu.emu_hyper_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), ctypes.c_int64(B), _p(n0), _p(n1),
                            _p(n2), _p(x), _p(ws))
    if running is not None:
        running.update({key: keep[key] for key in hu.RUNNING})
    return x, ws


def emu_bwd(emu, sd, e, r, B, gx, x, ws, n0=None, n1=None, n2=None):
    p, keep = hu.model_struct(sd, running=False)
    e, r, n0, n1, n2 = hu._i64(e), hu._i64(r), hu._f32(n0), hu._f32(n1), hu._f32(n2)
    grads = [np.zeros(np.shape(sd[key]), np.float32) for key in hu.PARAMS]
    arr = (ctypes.c_void_p * 12)(*[g.ctypes.data for g in grads])
    emu.emu_hyper_train_bwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B), _p(n0), _p(n1),
                            _p(n2), _p(hu._f32(gx)), _p(hu._f32(x)), arr, _p(ws))
    return grads


def _both_directions(g):
    """the tail and head rows of a golden case as one call of two groups, with the reference's noise"""
    B = len(g["h"])
    e, r = np.concatenate([g["h"], g["t"]]), np.concatenate([g["r"], g["r"]])
    nt, nh = hu.noises(g, "tail"), hu.noises(g, "head")
    nz = [None if a is None else np.concatenate([a, b]) for a, b in zip(nt, nh)]
    return e, r, B, nz


@pytest.mark.parametrize("name", hu.CASES)
def test_emulated_forward_equals_oracle_bitwise_on_goldens(emu, name):
    g = hu.load(name)
    sd = hu.state(g)
    e, r, B, nz = _both_directions(g)
    run_e, run_o = {}, {}
    x, _ = emu_fwd(emu, sd, e, r, B, *nz, running=run_e)
    want = hu.oracle_fwd(sd, e, r, B, *nz, running=run_o)
    assert _bits_equal(x, want)
    for key in hu.RUNNING:
        assert _bits_equal(run_e[key], run_o[key]), key
        assert np.abs(run_e[key] - g["sd_after_" + key]).max() < 1e-5, key   # = the reference's two forwards


@pytest.mark.parametrize("name", hu.CASES)
def test_emulated_backward_within_the_fp32_bound(emu, name):
    g = hu.load(name)
    sd = hu.state(g)
    e, r, B, nz = _both_directions(g)
    x, ws = emu_fwd(emu, sd, e, r, B, *nz)
    gx = np.random.RandomState(5).randn(len(e), x.shape[1]).astype(np.float32)
    got = emu_bwd(emu, sd, e, r, B, gx, x, ws, *nz)
    want, _ = hu.oracle_bwd64(sd, e, r, B, gx, *nz)
    scale = max(np.abs(w).max() for w in want)
    # each output is a sum of at most B * F fp32 terms per group; the fp32 arithmetic of the statistics and of every
    # BatchNorm backward adds relative rounding of order 2^-24 per step: 1e-4 of the output's largest magnitude bounds
    # them; bn0's affine parameters and fc.bias (true gradient ~0 in front of a training-mode BatchNorm with dropouts
    # 0) are held to the step's scale
    for key, a, b in zip(hu.PARAMS, got, want):
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max() + 1e-6 * scale, key
    assert not got[1][0].any()   # relation row 0 is in the batch: padding_idx, no gradient


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_hyper_train.cpp) -------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_hyper_train.cpp", name,
                           HEADERS + (os.path.join(emu_build.EMU, "emu_hyper_train.cpp"),),
                           extra=["-g", "-fsanitize=thread"] + extra, shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_hyper_train", [])
    probe = subprocess.run([exe, "probe"], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_hyper_train_kernels_are_race_free(race_checker):
    res = subprocess.run([race_checker], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_hyper_train -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_hyper_train_kernels(race_checker):
    """positive control: the same kernels with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_hyper_train_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
