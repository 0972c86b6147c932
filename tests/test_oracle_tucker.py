"""The TuckER oracle (tests/oracle_tucker/kge_oracle_tucker.c: core matrices per distinct relation, trunk forward in
the canonical summation orders, backward in double) against the reference's own outputs (tests/golden/tucker/) and
against fp64 autograd of the reference's per-sample formulation.  CPU only; the kernels are compared with this oracle
in tests/test_emu_tucker.py (emulated) and tests/test_gpu_tucker.py (on the device)."""
import numpy as np
import pytest
import torch

import golden_util as gu
import tucker_util as tu


def _preds(tabs, x):
    return 1.0 / (1.0 + np.exp(-(x.astype(np.float64) @ tabs[0].astype(np.float64).T)))


@pytest.mark.parametrize("name", tu.CASES)
def test_oracle_predictions_and_ranks_match_reference(name):
    g = tu.load(name)
    tabs = tu.tables(g)
    ids, slot = tu.slots(g["r"])
    assert len(ids) < len(g["r"]) and len(ids) < int(g["R"])   # relations repeat in the batch, others are absent
    M = tu.oracle_cores(tabs, ids)
    rows = g["query_rows"]
    ranks = np.zeros((len(rows), 4), dtype=np.int64)
    for d, (tag, e, tgt) in enumerate((("tail", g["h"], g["t"]), ("head", g["t"], g["h"]))):
        p = _preds(tabs, tu.oracle_trunk(tabs, M, e, slot)[0])
        assert gu.rel_err(p, g["preds_" + tag]).max() < 1e-4
        ptr, idx = g["filt_%s_ptr" % tag[0]], g["filt_%s_idx" % tag[0]]
        for qi, row in enumerate(rows):
            better = p[row] > p[row, tgt[row]]
            ranks[qi, 2 * d] = better.sum()
            known = idx[ptr[qi]:ptr[qi + 1]]
            ranks[qi, 2 * d + 1] = better.sum() - better[known[known != tgt[row]]].sum()
    assert int(g["n_ambiguous"]) == 0
    assert np.array_equal(ranks, g["ranks"])


@pytest.mark.parametrize("name", tu.CASES)
def test_oracle_loss_and_gradients_match_reference(name):
    """dropouts 0, or the reference's captured noise fed to the explicit mask mode"""
    g = tu.load(name)
    tabs = tu.tables(g)
    loss, grads, preds = tu.oracle_step(tabs, g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"],
                                        float(g["label_smoothing"]), tu.noises(g))
    assert gu.rel_err(preds[0], g["tr_preds_tail"]).max() < 1e-4
    assert gu.rel_err(preds[1], g["tr_preds_head"]).max() < 1e-4
    assert abs(loss - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    tu.golden_grad_check(g, grads, 5e-4)


def _autograd64(tabs, e, r, gx, noise0, m1, noise2):
    """fp64 autograd of the reference's formulation (one matrix per sample) -> (gent, grel, gW)"""
    ent, rel, W = [torch.tensor(t, dtype=torch.float64, requires_grad=True) for t in tabs]
    d1 = ent.shape[1]
    eh = torch.nn.functional.normalize(ent[torch.from_numpy(e)], p=2, dim=1)
    if noise0 is not None:
        eh = eh * torch.tensor(noise0, dtype=torch.float64)
    Wm = (rel[torch.from_numpy(r)] @ W).view(-1, d1, d1)
    if m1 is not None:
        Wm = Wm * torch.tensor(m1, dtype=torch.float64)
    x = torch.nn.functional.normalize(torch.matmul(eh.view(-1, 1, d1), Wm).view(-1, d1), p=2, dim=1)
    if noise2 is not None:
        x = x * torch.tensor(noise2, dtype=torch.float64)
    (x * torch.tensor(gx, dtype=torch.float64)).sum().backward()
    return [t.grad.numpy() for t in (ent, rel, W)]


@pytest.mark.parametrize("mode", ["none", "explicit", "counter"])
def test_oracle_backward_matches_fp64_autograd(mode):
    rng = np.random.RandomState(5)
    N, R, d1, d2, Q, p = 11, 6, 13, 5, 9, 0.4
    tabs = [rng.randn(N, d1).astype(np.float32), rng.randn(R, d2).astype(np.float32),
            rng.randn(d2, d1 * d1).astype(np.float32)]
    e, r = rng.randint(N, size=Q), rng.choice([4, 1, 2], size=Q)
    gx = rng.randn(Q, d1).astype(np.float32)
    noise0 = ((rng.rand(Q, d1) > 0.3) / 0.7).astype(np.float32)
    noise2 = ((rng.rand(Q, d1) > 0.5) / 0.5).astype(np.float32)
    mask, m1 = None, None
    if mode == "explicit":
        m1 = ((rng.rand(Q, d1, d1) > p) / (1 - p)).astype(np.float32)
        mask = ("explicit", m1)
    elif mode == "counter":
        mask = ("counter", 1234567, 40, p)
        m1 = tu.oracle_mask1(1234567, 40, p, Q, d1)
    ids, slot = tu.slots(r)
    M = tu.oracle_cores(tabs, ids)
    gent, dM = tu.oracle_trunk_bwd(tabs, M, e, slot, gx, noise0, mask, noise2)
    grel, gW = tu.oracle_cores_bwd(tabs, ids, dM)
    for got, want in zip((gent, grel, gW), _autograd64(tabs, e, r, gx, noise0, m1, noise2)):
        assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()   # M is rounded to fp32 once; the rest is fp64


def test_counter_mask_statistics():
    """kept fraction within binomial bounds of 1 - p, value 1 / (1 - p); (seed, offset) select the mask; element
    (q, i, j) is offset + its flat index, so a mask does not depend on how the queries are split over calls"""
    Q, d1, p = 6, 40, 0.3
    m = tu.oracle_mask1(99, 0, p, Q, d1)
    n = m.size
    assert set(np.unique(m)) == {np.float32(0.0), np.float32(1.0) / np.float32(0.7)}
    assert abs((m != 0).mean() - (1 - p)) < 5 * np.sqrt(p * (1 - p) / n)
    assert not np.array_equal(m, tu.oracle_mask1(100, 0, p, Q, d1))
    assert not np.array_equal(m, tu.oracle_mask1(99, 4, p, Q, d1))
    tail = tu.oracle_mask1(99, 2 * d1 * d1, p, Q - 2, d1)
    assert np.array_equal(m[2:], tail)
    assert np.all(tu.oracle_mask1(99, 0, 0.0, 2, d1) == 1.0) and np.all(tu.oracle_mask1(99, 0, 1.0, 2, d1) == 0.0)
