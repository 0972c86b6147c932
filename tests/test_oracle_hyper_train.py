"""The CPU oracle of HypER's training-mode trunk (tests/oracle_hyper_train) against the reference and against fp64
autograd, no GPU needed: the reference's training step (golden/hyper_train: the noise its dropout modules drew, loss,
every parameter's gradient, running statistics after both forwards) recomputed with the oracle's fp32 forward and fp64
backward, and the oracle's fp64 backward against torch fp64 autograd of the same formulas."""
import numpy as np
import pytest
import torch

import conve_train_util as cu
import hyper_train_util as hu


@pytest.mark.parametrize("name", hu.CASES)
def test_oracle_step_matches_reference(name):
    g = hu.load(name)
    loss, grads, run, xt, xh = hu.golden_step(g)
    assert abs(loss - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    for got, want in ((xt, g["x_tail"]), (xh, g["x_head"])):
        assert np.abs(got - want).max() <= 1e-5 * (1 + np.abs(want).max())
    cu.golden_grad_check(g, grads)
    # padding_idx = 0: relation row 0 (in the batch) gets no gradient; entity row 0 only the tail product's
    assert not grads["rel_embeddings.weight"][0].any() and grads["ent_embeddings.weight"][0].any()
    for key in hu.RUNNING:
        assert np.abs(run[key] - g["sd_after_" + key]).max() < 1e-5, key


def _torch64(sd, e, r, n0, n1, n2, pad):
    """the training-mode trunk (projection.py:581-606) in torch float64 with autograd on every trunk tensor"""
    P = [torch.tensor(np.asarray(sd[key], np.float64), requires_grad=True) for key in hu.PARAMS]
    ent, rel, w0, b0, w1, b1, fw, fb, w2, b2, f1w, f1b = P
    B, de = len(e), ent.shape[1]

    def bn(v, dims, w, b):
        mean = v.mean(dims, keepdim=True)
        return (v - mean) / torch.sqrt(v.var(dims, unbiased=False, keepdim=True) + 1e-5) * w + b

    et, rt = torch.from_numpy(e), torch.from_numpy(r)
    ev = torch.nn.functional.embedding(et, ent, padding_idx=pad)
    rv = torch.nn.functional.embedding(rt, rel, padding_idx=pad)
    x = bn(ev.view(B, 1, 1, de), (0, 1, 2, 3), w0.view(1, -1, 1, 1), b0.view(1, -1, 1, 1))
    x = x * torch.from_numpy(n0).double().view(B, 1, 1, de)
    k = (rv @ f1w.t() + f1b).view(B * 32, 1, 1, 9)
    x = torch.nn.functional.conv2d(x.permute(1, 0, 2, 3), k, groups=B).view(B, 32, 1, de - 8)
    x = bn(x, (0, 2, 3), w1.view(1, -1, 1, 1), b1.view(1, -1, 1, 1)) * torch.from_numpy(n1).double().view(B, 32, 1, 1)
    x = (x.reshape(B, -1) @ fw.t() + fb) * torch.from_numpy(n2).double()
    return torch.relu(bn(x, (0,), w2, b2)), P


@pytest.mark.parametrize("de,dr,B,G", [(24, 10, 5, 2), (17, 33, 3, 1)])
def test_oracle_backward_matches_fp64_autograd(de, dr, B, G):
    """random tables and noise, repeated ids and the padding id 0, G groups of B rows with their own statistics"""
    rng = np.random.RandomState(de + B)
    N, R, Q = 9, 4, G * B
    F = 32 * (de - 8)
    sd = {"ent_embeddings.weight": rng.randn(N, de), "rel_embeddings.weight": rng.randn(R, dr),
          "bn0.weight": rng.uniform(0.5, 1.5, 1), "bn0.bias": rng.uniform(-0.2, 0.2, 1),
          "bn1.weight": rng.uniform(0.5, 1.5, 32), "bn1.bias": rng.uniform(-0.2, 0.2, 32),
          "fc.weight": rng.randn(de, F) / np.sqrt(F), "fc.bias": 0.1 * rng.randn(de),
          "bn2.weight": rng.uniform(0.5, 1.5, de), "bn2.bias": rng.uniform(-0.2, 0.2, de),
          "fc1.weight": rng.randn(288, dr) / np.sqrt(dr), "fc1.bias": 0.1 * rng.randn(288)}
    sd = {key: v.astype(np.float32) for key, v in sd.items()}
    for key in hu.RUNNING:
        sd[key] = np.ones(1 if key.startswith("bn0") else (32 if key.startswith("bn1") else de), np.float32)
    e, r = rng.randint(N, size=Q), rng.randint(R, size=Q)
    e[1], r[2], e[0], r[1] = e[0], r[0], 0, 0
    n0 = ((rng.rand(Q, de) > 0.3) / np.float32(0.7)).astype(np.float32)
    n1 = ((rng.rand(Q, 32) > 0.2) / np.float32(0.8)).astype(np.float32)
    n2 = ((rng.rand(Q, de) > 0.3) / np.float32(0.7)).astype(np.float32)
    gx = rng.randn(Q, de)
    got, x64 = hu.oracle_bwd64(sd, e, r, B, gx, n0, n1, n2)
    want = [np.zeros(np.shape(sd[key])) for key in hu.PARAMS]
    for g0 in range(0, Q, B):
        s = slice(g0, g0 + B)
        x, P = _torch64(sd, e[s], r[s], n0[s], n1[s], n2[s], 0)
        assert np.abs(x.detach().numpy() - x64[s]).max() <= 1e-9 * (1 + np.abs(x64).max())
        (x * torch.from_numpy(gx[s])).sum().backward()
        for i, p in enumerate(P):
            want[i] += p.grad.numpy()
    for key, a, b in zip(hu.PARAMS, got, want):
        assert np.abs(a - b).max() <= 1e-8 * (1 + np.abs(b).max()), key
    assert not got[1][0].any()
    # the fp32 forward restates the same function
    x32 = hu.oracle_fwd(sd, e, r, B, n0, n1, n2)
    assert np.abs(x32 - x64).max() <= 1e-5 * (1 + np.abs(x64).max())
