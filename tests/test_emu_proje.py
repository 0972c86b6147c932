"""CPU check of ProjE_pointwise's CUDA kernels (pykg2vec_b200/csrc/kge_proje.cuh) under the host emulation
(tests/emu/cuda_runtime.h: every CUDA thread of a block is a host thread), with the launch geometry of the C-ABI
launchers: the trunk, the training step's per-entry logits and g, the negative labels and the L1 regulariser must
equal the oracle (tests/oracle_proje) bit for bit; the step's sums (loss, gradients) within fp32 reordering.
A ThreadSanitizer build of the step kernel (tests/emu/race_check_proje.cpp) checks its shared-memory
synchronisation; its barrier-free control build must be flagged.  The real kernels: tests/test_gpu_proje.py."""
import ctypes
import os
import subprocess

import numpy as np
import pytest

import emu_build
import proje_util as pu

HEADERS = ("kge_common.cuh", "kge_proj.cuh", "kge_proje.cuh")


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.build("emu_proje.cpp", "libemu_proje.so", HEADERS))


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _trunk(emu, tabs, e, r, d, noise=None):
    p, keep = pu.proje_struct(tabs)
    e, r = pu._i64(e), pu._i64(r)
    noise = pu._f32(noise)
    x = np.full((len(e), p.hidden_size), np.nan, dtype=np.float32)
    emu.emu_proje_trunk(ctypes.byref(p), d, _p(e), _p(r), ctypes.c_int64(len(e)), _p(noise), _p(x))
    return x


def _step(emu, tabs, h, r, t, lt, lh, nt=None, nh=None):
    p, keep = pu.proje_struct(tabs)
    h, r, t = pu._i64(h), pu._i64(r), pu._i64(t)
    lt, lh, nt, nh = pu._f32(lt), pu._f32(lh), pu._f32(nt), pu._f32(nh)
    B, N = len(r), p.num_ent
    grads = [np.zeros_like(a) for a in keep]
    gp = (ctypes.c_void_p * 8)(*[g.ctypes.data for g in grads])
    logit = np.full((2, B, N), np.nan, dtype=np.float32)
    gg = np.full((2, B, N), np.nan, dtype=np.float32)
    loss = np.zeros(1, dtype=np.float32)
    emu.emu_proje_step(ctypes.byref(p), _p(h), _p(r), _p(t), ctypes.c_int64(B), _p(lt), _p(lh), _p(nt), _p(nh), gp,
                       _p(loss), _p(logit), _p(gg))
    return float(loss[0]), grads, logit, gg


def _check_step(emu, tabs, h, r, t, lt, lh, nt=None, nh=None):
    loss, grads, logit, gg = _step(emu, tabs, h, r, t, lt, lh, nt, nh)
    wloss, wgrads, wlogit, wg = pu.oracle_step(tabs, h, r, t, lt, lh, nt, nh, per_entry=True)
    lab = np.stack([np.zeros_like(lt if lt is not None else lh) if a is None else a for a in (lt, lh)]) != 0
    assert _bits_equal(logit[lab], wlogit[lab]), "logits"
    assert _bits_equal(gg[lab], wg[lab]), "g"
    assert np.isnan(logit[~lab]).all(), "an entry with label 0 was evaluated"
    assert abs(loss - wloss) <= 1e-5 * abs(wloss)
    for key, a, b in zip(pu.KEYS, grads, wgrads):
        assert np.abs(a - b).max() <= 1e-5 * np.abs(b).max() + 1e-7, key
    return grads


@pytest.mark.parametrize("name", pu.CASES)
def test_emulated_trunk_bit_exact(emu, name):
    g = pu.load(name)
    tabs = pu.tables(pu.state(g))
    for d, (tag, e) in enumerate((("tail", g["h"]), ("head", g["t"]))):
        x = _trunk(emu, tabs, e, g["r"], d)
        assert _bits_equal(x, pu.oracle_trunk(tabs, e, g["r"], d))
        assert np.abs(x - g["x_" + tag]).max() <= 1e-6
        nz = g["noise_" + tag]
        assert _bits_equal(_trunk(emu, tabs, e, g["r"], d, nz), pu.oracle_trunk(tabs, e, g["r"], d, nz))


@pytest.mark.parametrize("name", pu.CASES)
def test_emulated_step_matches_oracle(emu, name):
    g = pu.load(name)
    tabs = pu.tables(pu.state(g))
    _check_step(emu, tabs, g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"], pu.noise_or_none(g, "tail"),
                pu.noise_or_none(g, "head"))


def test_emulated_step_flushes_long_label_rows(emu):
    """rows with more labelled entries than the list holds (2048): the list is processed mid-row; k = 18 takes the
    scalar (non-float4) logit loop; one direction only"""
    rng = np.random.RandomState(3)
    N, R, k, B = 5000, 4, 18, 3
    tabs = [rng.standard_normal((N, k)).astype(np.float32) * 0.3, rng.standard_normal((R, k)).astype(np.float32) * 0.3]
    tabs += [rng.standard_normal((1, k)).astype(np.float32) for _ in range(6)]
    lab = rng.choice(np.float32([-1, 0, 1, 0.5]), size=(B, N), p=[0.4, 0.2, 0.3, 0.1]).astype(np.float32)
    h, r, t = rng.randint(N, size=B), rng.randint(R, size=B), rng.randint(N, size=B)
    noise = (rng.rand(B, k) < 0.5).astype(np.float32) * 2
    grads = _check_step(emu, tabs, h, r, t, lab, None, noise, None)
    assert not grads[5].any() and not grads[6].any() and not grads[7].any()   # the head direction did not run


def test_emulated_negative_labels_rule(emu):
    rng = np.random.RandomState(0)
    B, N = 5, 300
    lab = (rng.rand(B, N) < 0.05).astype(np.float32)
    neg = rng.permutation(N)[:100].astype(np.int64)
    want = lab.copy()
    for b in range(B):
        for n in neg:
            if want[b, n] == 0:
                want[b, n] = -1.0
    emu.emu_labels_negatives(_p(lab), ctypes.c_int64(B), ctypes.c_int64(N), _p(neg), ctypes.c_int64(len(neg)))
    assert np.array_equal(lab, want)
    assert ((lab == -1).sum(axis=1) + (lab[:, neg] == 1).sum(axis=1) == 100).all()


def test_emulated_l1_regulariser(emu):
    rng = np.random.RandomState(1)
    ts = [rng.standard_normal(n).astype(np.float32) for n in (3000, 700, 16, 16)]
    ts[0][:10] = 0.0
    lm = np.float32(1e-3)
    grads = [rng.standard_normal(t.size).astype(np.float32) for t in ts]
    want = [g.copy() for g in grads]
    total = 0.0
    for t, w in zip(ts, want):
        total += pu.oracle_lib().kgeo_reg_l1(_p(t), ctypes.c_int64(t.size), ctypes.c_float(lm), _p(w))
    out = np.zeros(1, dtype=np.float32)
    wp = (ctypes.c_void_p * 4)(*[t.ctypes.data for t in ts])
    gp = (ctypes.c_void_p * 4)(*[g.ctypes.data for g in grads])
    ns = (ctypes.c_int64 * 4)(*[t.size for t in ts])
    emu.emu_reg_l1(wp, gp, ns, 4, ctypes.c_float(lm), _p(out))
    assert abs(float(out[0]) - total) <= 1e-5 * total
    for a, b in zip(grads, want):
        assert _bits_equal(a, b)


# ---- data-race check (ThreadSanitizer build of tests/emu/race_check_proje.cpp) ---------------------------
TSAN_ENV = dict(os.environ, TSAN_OPTIONS="exitcode=66 halt_on_error=1")


def _race_build(name, extra):
    return emu_build.build("race_check_proje.cpp", name, HEADERS, extra=["-g", "-fsanitize=thread"] + extra,
                           shared=False)


@pytest.fixture(scope="module")
def race_checker():
    exe = _race_build("race_check_proje", [])
    probe = subprocess.run([exe], env=TSAN_ENV, capture_output=True, text=True)
    if probe.returncode != 64:     # usage exit code: the sanitizer runtime itself starts up here
        pytest.skip("ThreadSanitizer runtime unavailable in this environment: %s" % probe.stderr[-300:])
    return exe


def test_proje_step_kernel_is_race_free(race_checker):
    res = subprocess.run([race_checker, "step"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 0, "race_check_proje step -> rc %d\n%s" % (res.returncode, res.stderr[-3000:])


def test_race_detector_flags_a_missing_barrier_in_the_proje_step(race_checker):
    """positive control: the same kernel with __syncthreads() compiled out must be reported"""
    exe = _race_build("race_check_proje_nobar", ["-DCUDA_EMU_NO_BARRIERS"])
    res = subprocess.run([exe, "step"], env=TSAN_ENV, capture_output=True, text=True, timeout=900)
    assert res.returncode == 66 and "data race" in res.stderr
