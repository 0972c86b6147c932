"""CPU check of AcrE's training-mode trunk kernels (pykg2vec_b200/csrc/kge_acre_train.cuh, the kge_conve_train.cuh
kernels and the tiled GEMM they launch) under the host emulation (tests/emu/cuda_runtime.h: every CUDA thread of a
block is a host thread), with the launch sequence of kge_acre_train_fwd / _bwd: x and the running statistics must equal
the oracle (tests/oracle_acre_train) bit for bit, the tail and head forwards as one call over two groups; the backward
agrees with the oracle's fp64 backward within the fp32 summation bound.  A ThreadSanitizer build
(tests/emu/race_check_acre_train.cpp) checks the shared-memory synchronisation of the CTA-per-query kernels; its
barrier-free control build must be flagged.  The real kernels: tests/test_gpu_acre_train.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import acre_train_util as atu
import emu_build

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_conve.cuh", "kge_conve_train.cuh", "kge_hyper.cuh", "kge_acre.cuh",
           "kge_acre_train.cuh")
_p = atu._p
# (way, C, atrous, acre_bias): small configurations of both ways, one with rates beyond the 20 x 20 image
CONFIGS = [("serial", 9, (1, 2, 3), True), ("parallel", 3, (2, 11, 23), False)]


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.build("emu_acre_train.cpp", "libemu_acre_train.so", HEADERS))


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def emu_fwd(emu, sd, e, r, B, n0=None, n1=None, n2=None, running=None):
    """the emulated forward -> (x, workspace); `running` (a dict) receives the updated running statistics"""
    p, keep = atu.model_struct(sd)
    e, r, n0, n1, n2 = atu._i64(e), atu._i64(r), atu._f32(n0), atu._f32(n1), atu._f32(n2)
    Q = len(e)
    emu.emu_acre_train_workspace_floats.restype = ctypes.c_int64
    ws = np.zeros(emu.emu_acre_train_workspace_floats(ctypes.byref(p), ctypes.c_int64(Q), ctypes.c_int64(B)),
                  np.float32)
    x = np.full((Q, 200), np.nan, np.float32)
    emu.emu_acre_train_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), ctypes.c_int64(B), _p(n0), _p(n1),
                           _p(n2), _p(x), _p(ws))
    if running is not None:
        running.update({key: keep[key] for key in atu.RUNNING})
    return x, ws


def emu_bwd(emu, sd, e, r, B, gx, x, ws, n0=None, n1=None, n2=None):
    p, keep = atu.model_struct(sd, running=False)
    e, r, n0, n1, n2 = atu._i64(e), atu._i64(r), atu._f32(n0), atu._f32(n1), atu._f32(n2)
    grads = {key: np.zeros(np.shape(sd[key]), np.float32) for key in atu.present(sd)}
    arr = (ctypes.c_void_p * len(atu.SLOTS))(*[grads[k].ctypes.data if k in grads else None for k in atu.SLOTS])
    emu.emu_acre_train_bwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(len(e)), ctypes.c_int64(B), _p(n0), _p(n1),
                           _p(n2), _p(atu._f32(gx)), _p(atu._f32(x)), arr, _p(ws))
    return [grads[k] for k in atu.present(sd)]


def _both_directions(g):
    """the tail and head rows of a golden case as one call of two groups, with the reference's noise"""
    B = len(g["h"])
    e, r = np.concatenate([g["h"], g["t"]]), np.concatenate([g["r"], g["r"]])
    nt, nh = atu.noises(g, "tail"), atu.noises(g, "head")
    nz = [None if a is None else np.concatenate([a, b]) for a, b in zip(nt, nh)]
    return e, r, B, nz


def _random_case(cfg, B=3, seed=4):
    rng = np.random.RandomState(seed)
    sd = atu.random_state(9, 4, cfg, seed)
    Q = 2 * B
    e, r = rng.randint(9, size=Q), rng.randint(8, size=Q)
    e[1], r[2], e[B] = e[0], r[0], e[0]
    nz = [((rng.rand(Q, w) > q) / np.float32(1 - q)).astype(np.float32) for w, q in ((400, 0.3), (cfg[1], 0.2),
                                                                                    (200, 0.5))]
    return sd, e, r, B, nz


@pytest.mark.parametrize("name", atu.CASES)
def test_emulated_forward_equals_oracle_bitwise_on_goldens(emu, name):
    g = atu.load(name)
    sd = atu.state(g)
    e, r, B, nz = _both_directions(g)
    run_e, run_o = {}, {}
    x, _ = emu_fwd(emu, sd, e, r, B, *nz, running=run_e)
    want = atu.oracle_fwd(sd, e, r, B, *nz, running=run_o)
    assert _bits_equal(x, want)
    for key in atu.RUNNING:
        assert _bits_equal(run_e[key], run_o[key]), key
        assert np.abs(run_e[key] - g["sd_after_" + key]).max() < 1e-5, key   # = the reference's two forwards


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: c[0])
def test_emulated_forward_equals_oracle_bitwise_with_noise(emu, cfg):
    sd, e, r, B, nz = _random_case(cfg)
    run_e, run_o = {}, {}
    x, _ = emu_fwd(emu, sd, e, r, B, *nz, running=run_e)
    assert _bits_equal(x, atu.oracle_fwd(sd, e, r, B, *nz, running=run_o))
    assert all(_bits_equal(run_e[key], run_o[key]) for key in atu.RUNNING)


def _check_bwd(emu, sd, e, r, B, nz):
    x, ws = emu_fwd(emu, sd, e, r, B, *nz)
    gx = np.random.RandomState(5).randn(len(e), 200).astype(np.float32)
    got = emu_bwd(emu, sd, e, r, B, gx, x, ws, *nz)
    want, _ = atu.oracle_bwd64(sd, e, r, B, gx, *nz)
    scale = max(np.abs(w).max() for w in want)
    # each output is a sum of at most B * C * 400 * 9 fp32 terms per group; the fp32 arithmetic of the statistics and
    # of every BatchNorm backward adds relative rounding of order 2^-24 per step: 1e-4 of the output's largest
    # magnitude bounds them; sums that cancel to a small result (the biases in front of a training-mode BatchNorm,
    # whose true gradient is ~0, and bn0's affine parameters, sums over 2 * B * 400 terms of both signs) are held to
    # 1e-5 of the step's scale
    for key, a, b in zip(atu.present(sd), got, want):
        assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max() + 1e-5 * scale, key


@pytest.mark.parametrize("name", atu.CASES)
def test_emulated_backward_within_the_fp32_bound_on_goldens(emu, name):
    g = atu.load(name)
    _check_bwd(emu, atu.state(g), *_both_directions(g))


@pytest.mark.parametrize("cfg", CONFIGS, ids=lambda c: c[0])
def test_emulated_backward_within_the_fp32_bound_with_noise(emu, cfg):
    _check_bwd(emu, *_random_case(cfg))


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_acre_train.cpp) -----------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_acre_train.cpp", name,
                           HEADERS + (os.path.join(emu_build.EMU, "emu_acre_train.cpp"),),
                           extra=["-g", "-fsanitize=thread"] + extra, shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_acre_train", [])
    probe = subprocess.run([exe, "probe"], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_acre_train_kernels_are_race_free(race_checker):
    res = subprocess.run([race_checker], env=TSAN_ENV, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 0, "race_check_acre_train -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_acre_train_kernels(race_checker):
    """positive control: the same kernels with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_acre_train_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True, timeout=1200)
    assert res.returncode == 66 and "data race" in res.stderr
