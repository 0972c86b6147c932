"""CPU check of InteractE's inference-trunk CUDA kernels (pykg2vec_b200/csrc/kge_interacte.cuh) under the host
emulation (tests/emu/cuda_runtime.h: every CUDA thread of a block is a host thread), through the same workspace
layout and launch plans as the C-ABI launcher: the features (gather + chequer permutation + bn0 + circular conv
+ bn1 + ReLU), the sliced Linear GEMM and the bn2 + ReLU combine must equal the oracle bit for bit — on the
reference's own parameters and at the largest yaml configuration, (P, F, ks) = (4, 64, 7) on a 20 x 10 reshape.
A ThreadSanitizer build of the feature kernel (tests/emu/race_check_interacte.cpp) checks its shared-memory
synchronisation; its barrier-free control build must be flagged.
The real kernels are checked on the GPU by tests/test_gpu_interacte.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import emu_build
import interacte_util as iu

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_conve.cuh", "kge_hyper.cuh", "kge_interacte.cuh")


@pytest.fixture(scope="module")
def emu():
    L = ctypes.CDLL(emu_build.build("emu_interacte.cpp", "libemu_interacte.so", HEADERS))
    L.emu_interacte_workspace_floats.restype = ctypes.c_int64
    L.emu_interacte_smem_bytes.restype = ctypes.c_int64
    return L


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _run(emu, st, perm, e, r):
    """-> (x, features) of the emulated kernels"""
    p, keep = iu.interacte_struct(st, perm)
    e, r = np.ascontiguousarray(e, dtype=np.int64), np.ascontiguousarray(r, dtype=np.int64)
    Q, k = len(e), p.reshape_height * p.reshape_width
    ws = np.full(emu.emu_interacte_workspace_floats(ctypes.byref(p), ctypes.c_int64(Q)), np.nan, dtype=np.float32)
    x = np.full((Q, k), np.nan, dtype=np.float32)
    assert emu.emu_interacte_trunk_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), _p(x), _p(ws)) == 0
    Fw = p.feature_permutation * p.num_filters * 2 * k
    return x, ws[:Q * Fw].reshape(Q, Fw)


def _bits_equal(a, b):
    return np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("name", iu.CASES)
def test_emulated_trunk_bit_exact_on_reference_parameters(emu, name):
    g = iu.load(name)
    st = iu.state(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        x, feat = _run(emu, st, g["chequer_perm"], e, g["r"])
        wx, wfeat = iu.oracle_trunk_fwd(st, g["chequer_perm"], e, g["r"], intermediates=True)
        assert _bits_equal(feat, wfeat), "feature kernel"
        assert _bits_equal(x, wx), "Linear + combine"
        assert np.abs(x - g["x_" + tag]).max() <= 1e-5


def test_emulated_trunk_bit_exact_at_largest_yaml_config(emu):
    """(P, F, ks, rh, rw) = (4, 64, 7, 20, 10): 200 Linear slices of 512 features, Q = 33"""
    geom, N, R, Q = (4, 64, 7, 20, 10), 300, 237, 33
    st, perm = iu.random_state(N, R, geom, seed=47)
    rng = np.random.RandomState(5)
    e, r = rng.randint(N, size=Q), rng.randint(R, size=Q)
    e[:3], r[:3] = 0, 0
    x, feat = _run(emu, st, perm, e, r)
    wx, wfeat = iu.oracle_trunk_fwd(st, perm, e, r, intermediates=True)
    assert _bits_equal(feat, wfeat) and _bits_equal(x, wx)
    assert (x > 0).any() and (x == 0).any() and (feat == 0).any()       # both ReLUs are live


def test_shared_memory_of_the_yaml_configs(emu):
    """every yaml configuration fits the 227 KB per-block bound; (2, 96, 11) needs the opt-in above 48 KB"""
    sizes = {}
    for geom in iu.YAML_CONFIGS:
        st, perm = iu.random_state(4, 2, geom, seed=1)
        p, keep = iu.interacte_struct(st, perm)
        sizes[geom[:3]] = emu.emu_interacte_smem_bytes(ctypes.byref(p))
    assert all(s <= 227 * 1024 for s in sizes.values())
    assert sizes[(2, 96, 11)] > 48 * 1024


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_interacte.cpp) -----------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_interacte.cpp", name, HEADERS, extra=["-g", "-fsanitize=thread"] + extra,
                           shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_interacte", [])
    probe = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_interacte_feature_kernel_is_race_free(race_checker):
    res = subprocess.run([race_checker, "features"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_interacte features -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_interacte_kernel(race_checker):
    """positive control: the same kernel with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_interacte_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe, "features"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
