"""CPU check of the projection-tail CUDA kernels' LOGIC (no GPU in the build container).

pykg2vec_b200/csrc/kge_proj.cuh is compiled with g++ against tests/emu/cuda_runtime.h, which runs
every CUDA thread of a block as a host thread (barrier = __syncthreads, lane exchange =
__shfl_xor_sync, host atomics), through the same launch plans the C-ABI launchers use.  What this
pins before the GPU run: tiling and strides of the three GEMM uses, zero padding, split-K
ranges, the half-warp count reduction, the filter correction and the BCE reduction — against the
oracle (bit-exact where the arithmetic is canonical, tolerance where the summation order is free).
The real kernels are checked on the GPU by tests/test_gpu_proj.py."""
import ctypes
import os

import numpy as np
import pytest

import oracle

import emu_build
import golden_util as gu

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu():
    return ctypes.CDLL(emu_build.proj_lib())


def _p(a):
    return a.ctypes.data_as(ctypes.c_void_p) if a is not None else None


def _case(B, N, k, seed, bias=True):
    rng = np.random.RandomState(seed)
    x = np.maximum(rng.standard_normal((B, k)) * 0.7, 0).astype(np.float32)   # post-ReLU operand
    ent = (rng.standard_normal((N, k)) * 0.5).astype(np.float32)
    b = (rng.standard_normal(N) * 0.3).astype(np.float32) if bias else None
    return x, ent, b


SHAPES = [(70, 131, 48, True), (5, 64, 50, True), (64, 65, 7, False), (1, 200, 16, True), (33, 1, 100, False)]


@pytest.mark.parametrize("tile", [0, 1, 2], ids=["64x64", "64x128", "128x128"])
@pytest.mark.parametrize("B,N,k,bias", SHAPES + [(130, 140, 20, True)])
def test_emulated_forward_is_bit_exact(emu, B, N, k, bias, tile):
    x, ent, b = _case(B, N, k, seed=B * 1000 + N, bias=bias)
    got = np.full((B, N), np.nan, dtype=np.float32)
    emu.emu_proj_tail_fwd(_p(x), _p(ent), _p(b), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k), _p(got),
                          ctypes.c_int32(tile))
    want = oracle.proj_tail_fwd(x, ent, b)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))


def test_emulated_forward_unaligned_operands(emu):
    """operands that are not 16-byte aligned must take the scalar loader and give the same bits"""
    B, N, k = 9, 77, 48
    x, ent, b = _case(B, N, k, seed=5)
    xb = np.zeros(B * k + 1, dtype=np.float32)
    xo = xb[1:].reshape(B, k)
    xo[:] = x
    assert xo.ctypes.data % 16 != 0
    got = np.empty((B, N), dtype=np.float32)
    emu.emu_proj_tail_fwd(_p(xo), _p(ent), _p(b), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k), _p(got),
                          ctypes.c_int32(2))
    assert np.array_equal(got, oracle.proj_tail_fwd(x, ent, b))


@pytest.mark.parametrize("tile", [0, 1, 2], ids=["64x64", "64x128", "128x128"])
@pytest.mark.parametrize("B,N,k,bias", SHAPES[:4] + [(130, 140, 20, True)])
def test_emulated_rank_counts(emu, B, N, k, bias, tile):
    x, ent, b = _case(B, N, k, seed=B * 77 + N, bias=bias)
    rng = np.random.RandomState(B + N)
    tgt = rng.randint(N, size=B).astype(np.int64)
    ptr = np.zeros(B + 1, dtype=np.int64)
    rows = []
    for q in range(B):
        n = rng.randint(0, min(N, 9))
        row = rng.choice(N, size=n, replace=False)
        if q % 2 == 0 and n:
            row[0] = tgt[q]            # the target itself appears in its filter row (hr_t contains t)
        rows.append(np.unique(row))
        ptr[q + 1] = ptr[q] + len(rows[-1])
    idx = np.concatenate(rows).astype(np.int64) if ptr[-1] else np.zeros(0, dtype=np.int64)
    for direction in (0, 1):
        got = np.zeros((B, 4), dtype=np.int32)
        thr = np.zeros(B, dtype=np.float32)
        emu.emu_proj_rank(_p(x), _p(ent), _p(b), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k), _p(tgt),
                          _p(ptr), _p(idx), ctypes.c_int64(len(idx)), ctypes.c_int32(direction), _p(got), _p(thr),
                          ctypes.c_int32(tile))
        want = oracle.proj_rank(x, ent, b, tgt, (ptr, idx), direction)
        assert np.array_equal(got, want)
        # and the counts are what counting over the forward matrix gives
        preds = oracle.proj_tail_fwd(x, ent, b)
        raw = (preds > preds[np.arange(B), tgt][:, None]).sum(1)
        assert np.array_equal(got[:, 2 * direction], raw)


@pytest.mark.parametrize("B,N,k,ctas", [(70, 131, 48, 12), (5, 300, 50, 296), (64, 65, 7, 1), (20, 97, 100, 7)])
def test_emulated_backward(emu, B, N, k, ctas):
    x, ent, b = _case(B, N, k, seed=B + 3 * N)
    rng = np.random.RandomState(k)
    preds = oracle.proj_tail_fwd(x, ent, b)
    gp = (rng.standard_normal((B, N)) * 0.1).astype(np.float32)
    gx = np.zeros((B, k), dtype=np.float32)
    ge = np.full((N, k), 0.25, dtype=np.float32)       # accumulate semantics: pre-filled
    gb = np.full(N, -0.5, dtype=np.float32)
    emu.emu_proj_tail_bwd(_p(gp), _p(preds), _p(x), _p(ent), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k),
                          _p(gx), _p(ge), _p(gb), ctypes.c_int32(ctas))
    wx, we, wb = oracle.proj_tail_bwd(gp, preds, x, ent)
    for got, want in ((gx, wx), (ge - 0.25, we), (gb + 0.5, wb)):
        assert np.abs(got - want).max() <= 2e-6 * max(1.0, np.abs(want).max())


@pytest.mark.parametrize("B,N,sms", [(7, 131, 148), (64, 300, 1), (3, 5, 148)])
def test_emulated_bce(emu, B, N, sms):
    rng = np.random.RandomState(B * N)
    preds = (1.0 / (1.0 + np.exp(-rng.standard_normal((B, N)) * 3))).astype(np.float32)
    labels = (rng.rand(B, N) < 0.1).astype(np.float32)
    scale, shift = np.float32(1.0 - 0.1), np.float32(1.0 / N)
    loss = np.zeros(1, dtype=np.float32)
    g = np.empty((B, N), dtype=np.float32)
    emu.emu_proj_bce(_p(preds), _p(labels), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_float(scale),
                     ctypes.c_float(shift), ctypes.c_float(1.0), _p(loss), _p(g), ctypes.c_int32(sms))
    want_loss, want_g = oracle.proj_bce(preds, labels, scale, shift, 1.0)
    assert abs(loss[0] - want_loss) <= 2e-6 * abs(want_loss)
    assert np.array_equal(g.view(np.uint32), want_g.view(np.uint32))


@pytest.mark.parametrize("name,Q", [("conve_d48", 7), ("conve_d100", 3)])
def test_emulated_conve_trunk(emu, name, Q):
    """gather + bn0 + conv + bn1 + relu kernel and the Linear GEMM, on the reference's own ConvE
    parameters: bit-exact vs the oracle, which is pinned on the reference's x (test_oracle_proj)."""
    g = gu.load(name)
    state = gu.proj_state(g)
    k, k1, R = int(g["hidden_size"]), int(g["hidden_size_1"]), int(g["R"])
    keep = {f: np.ascontiguousarray(state[key], dtype=np.float32) for f, key in oracle.CONVE_KEYS.items()}
    p = oracle.KgeConve()
    p.hidden_size, p.hidden_size_1, p.bn0_eps, p.bn1_eps = k, k1, 1e-5, 1e-5
    for f, a in keep.items():
        setattr(p, f, a.ctypes.data)
    e = np.ascontiguousarray(g["t"][:Q])
    r = np.ascontiguousarray(g["r"][:Q] + R)     # head direction: reciprocal relation ids
    F = 32 * (2 * (k // k1) - 2) * (k1 - 2)
    x = np.full((Q, k), np.nan, dtype=np.float32)
    feat = np.empty(Q * F + ((F + 511) // 512) * Q * k, dtype=np.float32)   # workspace: features + slice partials
    emu.emu_conve_trunk_fwd(ctypes.byref(p), _p(e), _p(r), ctypes.c_int64(Q), _p(x), _p(feat))
    want = oracle.conve_trunk_fwd(state, k, k1, e, r)
    assert np.array_equal(x.view(np.uint32), want.view(np.uint32))
    assert np.abs(x - g["x_head"][:Q]).max() <= 1e-5


@pytest.mark.parametrize("with_rows", [False, True])
def test_emulated_label_rows(emu, with_rows):
    rng = np.random.RandomState(9)
    K, N, B = 11, 300, 7
    sizes = rng.randint(0, 200, size=K)
    sizes[3] = 0
    ptr = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int64)
    idx = np.concatenate([rng.choice(N, size=n, replace=False) for n in sizes]).astype(np.int64)
    rows = rng.randint(K, size=B).astype(np.int64) if with_rows else None
    if not with_rows:
        B = K
    got = np.full((B, N), np.nan, dtype=np.float32)
    emu.emu_proj_labels(_p(rows), _p(ptr), _p(idx), ctypes.c_int64(B), ctypes.c_int64(N), _p(got))
    want = np.zeros((B, N), dtype=np.float32)
    for b in range(B):
        row = rows[b] if with_rows else b
        want[b, idx[ptr[row]:ptr[row + 1]]] = 1.0
    assert np.array_equal(got, want)


def test_emulated_random_shapes(emu):
    """seeded sweep over awkward shapes (1-wide operands, sizes straddling the 64 / 128 tile edges and the
    16-deep k chunks, every CTA tile): forward bits, rank counts and gradients against the oracle"""
    rng = np.random.RandomState(1234)
    edges = [1, 2, 15, 16, 17, 63, 64, 65, 127, 128, 129, 130]
    for it in range(10):
        B, N, k = int(rng.choice(edges)), int(rng.choice(edges)), int(rng.choice([1, 3, 4, 15, 16, 17, 33, 48]))
        tile = it % 3
        x, ent, b = _case(B, N, k, seed=it, bias=bool(it % 2))
        got = np.full((B, N), np.nan, dtype=np.float32)
        emu.emu_proj_tail_fwd(_p(x), _p(ent), _p(b), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k), _p(got),
                              ctypes.c_int32(tile))
        want = oracle.proj_tail_fwd(x, ent, b)
        assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), (B, N, k, tile)
        tgt = rng.randint(N, size=B).astype(np.int64)
        counts = np.zeros((B, 4), dtype=np.int32)
        thr = np.zeros(B, dtype=np.float32)
        emu.emu_proj_rank(_p(x), _p(ent), _p(b), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k), _p(tgt),
                          None, None, ctypes.c_int64(0), ctypes.c_int32(1), _p(counts), _p(thr), ctypes.c_int32(tile))
        assert np.array_equal(counts, oracle.proj_rank(x, ent, b, tgt, None, 1)), (B, N, k, tile)
        gp = (rng.standard_normal((B, N)) * 0.1).astype(np.float32)
        gx, ge, gb = np.zeros((B, k), np.float32), np.zeros((N, k), np.float32), np.zeros(N, np.float32)
        emu.emu_proj_tail_bwd(_p(gp), _p(want), _p(x), _p(ent), ctypes.c_int64(B), ctypes.c_int64(N), ctypes.c_int32(k),
                              _p(gx), _p(ge), _p(gb), ctypes.c_int32(int(rng.choice([1, 5, 296]))))
        wx, we, wb = oracle.proj_tail_bwd(gp, want, x, ent)
        for a, w in ((gx, wx), (ge, we), (gb, wb)):
            assert np.abs(a - w).max() <= 2e-6 * max(1.0, np.abs(w).max()), (B, N, k)
