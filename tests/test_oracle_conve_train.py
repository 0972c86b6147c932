"""The CPU oracle of ConvE's training-mode trunk (tests/oracle_conve_train) against the reference and against fp64
autograd, no GPU needed: the reference's training step (golden/conve_train: the noise its dropout modules drew, loss,
every parameter's gradient, running statistics after both forwards) recomputed with the oracle's fp32 forward and fp64
backward, and the oracle's fp64 backward against torch fp64 autograd of the same formulas."""
import numpy as np
import pytest
import torch

import conve_train_util as cu


@pytest.mark.parametrize("name", cu.CASES)
def test_oracle_step_matches_reference(name):
    g = cu.load(name)
    loss, grads, run, xt, xh = cu.golden_step(g)
    assert abs(loss - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    for got, want in ((xt, g["x_tail"]), (xh, g["x_head"])):
        assert np.abs(got - want).max() <= 1e-5 * (1 + np.abs(want).max())
    cu.golden_grad_check(g, grads)
    for key in cu.RUNNING:
        assert np.abs(run[key] - g["sd_after_" + key]).max() < 1e-5, key


def _torch64(sd, k, h1, e, r, n0, n1, n2):
    """the training-mode trunk (projection.py:86-99) in torch float64 with autograd on every trunk tensor"""
    P = [torch.tensor(np.asarray(sd[key], np.float64), requires_grad=True) for key in cu.PARAMS]
    ent, rel, w0, b0, cw, cb, w1, b1, fw, fb, w2, b2 = P
    B, h2 = len(e), k // h1

    def bn(v, dims, w, b):
        mean = v.mean(dims, keepdim=True)
        return (v - mean) / torch.sqrt(v.var(dims, unbiased=False, keepdim=True) + 1e-5) * w + b

    x = torch.cat([ent[torch.from_numpy(e)], rel[torch.from_numpy(r)]], 1).view(B, 1, 2 * h2, h1)
    x = bn(x, (0, 1, 2, 3), w0.view(1, -1, 1, 1), b0.view(1, -1, 1, 1)) * torch.from_numpy(n0).double().view(B, 1, 2 * h2, h1)
    x = torch.nn.functional.conv2d(x, cw, cb)
    x = torch.relu(bn(x, (0, 2, 3), w1.view(1, -1, 1, 1), b1.view(1, -1, 1, 1))) * torch.from_numpy(n1).double().view(B, 32, 1, 1)
    x = (x.reshape(B, -1) @ fw.t() + fb) * torch.from_numpy(n2).double()
    return torch.relu(bn(x, (0,), w2, b2)), P


@pytest.mark.parametrize("k,h1,B,G", [(36, 6, 5, 2), (20, 4, 3, 1)])
def test_oracle_backward_matches_fp64_autograd(k, h1, B, G):
    """random tables and noise, repeated ids, G groups of B rows with their own statistics"""
    rng = np.random.RandomState(k + B)
    N, R, Q = 9, 4, G * B
    F = 32 * (2 * (k // h1) - 2) * (h1 - 2)
    sd = {"ent_embeddings.weight": rng.randn(N, k), "rel_embeddings.weight": rng.randn(2 * R, k),
          "bn0.weight": rng.uniform(0.5, 1.5, 1), "bn0.bias": rng.uniform(-0.2, 0.2, 1),
          "conv2d_1.weight": 0.3 * rng.randn(32, 1, 3, 3), "conv2d_1.bias": 0.1 * rng.randn(32),
          "bn1.weight": rng.uniform(0.5, 1.5, 32), "bn1.bias": rng.uniform(-0.2, 0.2, 32),
          "fc.weight": rng.randn(k, F) / np.sqrt(F), "fc.bias": 0.1 * rng.randn(k),
          "bn2.weight": rng.uniform(0.5, 1.5, k), "bn2.bias": rng.uniform(-0.2, 0.2, k)}
    sd = {key: v.astype(np.float32) for key, v in sd.items()}
    for key in cu.RUNNING:
        sd[key] = np.ones(1 if key.startswith("bn0") else (32 if key.startswith("bn1") else k), np.float32)
    e, r = rng.randint(N, size=Q), rng.randint(2 * R, size=Q)
    e[1], r[2] = e[0], r[0]
    n0 = ((rng.rand(Q, 2 * k) > 0.2) / np.float32(0.8)).astype(np.float32)
    n1 = ((rng.rand(Q, 32) > 0.2) / np.float32(0.8)).astype(np.float32)
    n2 = ((rng.rand(Q, k) > 0.3) / np.float32(0.7)).astype(np.float32)
    gx = rng.randn(Q, k)
    got, x64 = cu.oracle_bwd64(sd, k, h1, e, r, B, gx, n0, n1, n2)
    want = [np.zeros(np.shape(sd[key])) for key in cu.PARAMS]
    for g0 in range(0, Q, B):
        s = slice(g0, g0 + B)
        x, P = _torch64(sd, k, h1, e[s], r[s], n0[s], n1[s], n2[s])
        assert np.abs(x.detach().numpy() - x64[s]).max() <= 1e-9 * (1 + np.abs(x64).max())
        (x * torch.from_numpy(gx[s])).sum().backward()
        for i, p in enumerate(P):
            want[i] += p.grad.numpy()
    for key, a, b in zip(cu.PARAMS, got, want):
        assert np.abs(a - b).max() <= 1e-8 * (1 + np.abs(b).max()), key
    # the fp32 forward restates the same function
    x32 = cu.oracle_fwd(sd, k, h1, e, r, B, n0, n1, n2)
    assert np.abs(x32 - x64).max() <= 1e-5 * (1 + np.abs(x64).max())
