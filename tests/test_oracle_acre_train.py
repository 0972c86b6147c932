"""The CPU oracle of AcrE's training-mode trunk (tests/oracle_acre_train) against the reference and against fp64
autograd, no GPU needed: the reference's training step (golden/acre_train: the noise its dropout modules drew, loss,
every parameter's gradient, running statistics after both forwards) recomputed with the oracle's fp32 forward and fp64
backward, and the oracle's fp64 backward against torch fp64 autograd of the same formulas, in both ways."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import acre_train_util as atu
import conve_train_util as cu


@pytest.mark.parametrize("name", atu.CASES)
def test_oracle_step_matches_reference(name):
    g = atu.load(name)
    loss, grads, run, xt, xh = atu.golden_step(g)
    assert abs(loss - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    for got, want in ((xt, g["x_tail"]), (xh, g["x_head"])):
        assert np.abs(got - want).max() <= 1e-5 * (1 + np.abs(want).max())
    # with dropouts 0, fc.bias (no ReLU between fc and bn2) and the conv / gate biases sit in front of a training-mode
    # BatchNorm: their true gradient is 0 and the reference's fp32 value is rounding noise of ~2e-7
    cu.golden_grad_check(g, grads, floor=1e-6)
    for key in atu.RUNNING:
        assert np.abs(run[key] - g["sd_after_" + key]).max() < 1e-5, key


def _torch64(sd, e, r, n0, n1, n2):
    """the training-mode trunk (projection.py:708-734) in torch float64 with autograd on every present trunk tensor"""
    way, C, rates = atu.config(sd)
    keys = atu.present(sd)
    T = {key: torch.tensor(np.asarray(sd[key], np.float64), requires_grad=True) for key in keys}
    B = len(e)

    def bn(v, dims, w, b):
        mean = v.mean(dims, keepdim=True)
        return (v - mean) / torch.sqrt(v.var(dims, unbiased=False, keepdim=True) + 1e-5) * w + b

    def conv(l, x):
        return F.conv2d(x, T["conv%d.weight" % l], T.get("conv%d.bias" % l), 1, rates[l - 1], rates[l - 1])

    img = torch.cat([T["ent_embeddings.weight"][torch.from_numpy(e)], T["rel_embeddings.weight"][torch.from_numpy(r)]],
                    1).view(B, 1, 20, 20)
    v = bn(img, (0, 2, 3), T["bn0.weight"].view(1, -1, 1, 1), T["bn0.bias"].view(1, -1, 1, 1))
    v = v * torch.from_numpy(n0).double().view(B, 1, 20, 20)
    if way == 0:
        y = conv(3, conv(2, conv(1, v))) + v
    else:
        gate = torch.cat([v.expand(-1, C, 20, 20).reshape(B, C, 400)] +
                         [conv(l, v).reshape(B, C, 400) for l in (1, 2, 3)], 2)
        y = (gate @ T["W_gate_e.weight"].t() + T["W_gate_e.bias"]).view(B, C, 20, 20)
    x = torch.relu(bn(y, (0, 2, 3), T["bn1.weight"].view(1, -1, 1, 1), T["bn1.bias"].view(1, -1, 1, 1)))
    x = x * torch.from_numpy(n1).double().view(B, C, 1, 1)
    x = (x.reshape(B, -1) @ T["fc.weight"].t() + T["fc.bias"]) * torch.from_numpy(n2).double()
    return torch.relu(bn(x, (0,), T["bn2.weight"], T["bn2.bias"])), [T[k] for k in keys]


@pytest.mark.parametrize("cfg,B,G", [(("serial", 3, (1, 2, 3), True), 4, 2), (("parallel", 2, (2, 11, 23), False), 3, 2),
                                     (("parallel", 3, (1, 1, 2), True), 5, 1), (("serial", 2, (3, 21, 1), False), 4, 1)])
def test_oracle_backward_matches_fp64_autograd(cfg, B, G):
    """random tables and noise, repeated ids, G groups of B rows with their own statistics, both ways"""
    rng = np.random.RandomState(B + 10 * G + cfg[1])
    N, R, Q = 9, 4, G * B
    sd = atu.random_state(N, R, cfg, seed=B + G)
    e, r = rng.randint(N, size=Q), rng.randint(2 * R, size=Q)
    e[1], r[-1] = e[0], r[0]
    n0 = ((rng.rand(Q, 400) > 0.3) / np.float32(0.7)).astype(np.float32)
    n1 = ((rng.rand(Q, cfg[1]) > 0.2) / np.float32(0.8)).astype(np.float32)
    n2 = ((rng.rand(Q, 200) > 0.3) / np.float32(0.7)).astype(np.float32)
    gx = rng.randn(Q, 200)
    got, x64 = atu.oracle_bwd64(sd, e, r, B, gx, n0, n1, n2)
    want = [np.zeros(np.shape(sd[key])) for key in atu.present(sd)]
    for g0 in range(0, Q, B):
        s = slice(g0, g0 + B)
        x, Pt = _torch64(sd, e[s], r[s], n0[s], n1[s], n2[s])
        assert np.abs(x.detach().numpy() - x64[s]).max() <= 1e-9 * (1 + np.abs(x64).max())
        (x * torch.from_numpy(gx[s])).sum().backward()
        for i, p in enumerate(Pt):
            want[i] += p.grad.numpy()
    for key, a, b in zip(atu.present(sd), got, want):
        assert np.abs(a - b).max() <= 1e-8 * (1 + np.abs(b).max()), key
    # the fp32 forward restates the same function
    x32 = atu.oracle_fwd(sd, e, r, B, n0, n1, n2)
    assert np.abs(x32 - x64).max() <= 1e-4 * (1 + np.abs(x64).max())
