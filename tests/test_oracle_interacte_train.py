"""The CPU oracle of InteractE's training-mode trunk (tests/oracle_interacte_train) against the reference and against
fp64 autograd, no GPU needed: the reference's training step (golden/interacte_train: the noise its dropout modules
drew, loss, every parameter's gradient, running statistics after both forwards) recomputed with the oracle's fp32
forward and fp64 backward, and the oracle's fp64 backward against torch fp64 autograd of the same formulas."""
import numpy as np
import pytest
import torch

import conve_train_util as cu
import interacte_train_util as itu


@pytest.mark.parametrize("name", itu.CASES)
def test_oracle_step_matches_reference(name):
    g = itu.load(name)
    loss, grads, run, xt, xh = itu.golden_step(g)
    assert abs(loss - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    for got, want in ((xt, g["x_tail"]), (xh, g["x_head"])):
        assert np.abs(got - want).max() <= 1e-5 * (1 + np.abs(want).max())
    cu.golden_grad_check(g, grads)
    for key in itu.RUNNING:
        assert np.abs(run[key] - g["sd_after_" + key]).max() < 1e-5, key


def _torch64(sd, e, r, n0, n1, n2):
    """the training-mode trunk (projection.py:427-442) in torch float64 with autograd on every trunk tensor"""
    P_, F_, ks, rh, rw = (int(v) for v in sd["_geometry"])
    H, W, pad = 2 * rw, rh, ks // 2
    P = [torch.tensor(np.asarray(sd[key], np.float64), requires_grad=True) for key in itu.PARAMS]
    ent, rel, w0, b0, filt, w1, b1, fw, fb, w2, b2 = P
    B = len(e)

    def bn(v, dims, w, b):
        mean = v.mean(dims, keepdim=True)
        return (v - mean) / torch.sqrt(v.var(dims, unbiased=False, keepdim=True) + 1e-5) * w + b

    comb = torch.cat([ent[torch.from_numpy(e)], rel[torch.from_numpy(r)]], dim=1)
    x = comb[:, torch.from_numpy(sd["_perm"])].reshape(B, P_, H, W)
    x = bn(x, (0, 2, 3), w0.view(1, -1, 1, 1), b0.view(1, -1, 1, 1)) * torch.from_numpy(n0).double().view(B, P_, H, W)
    x = torch.cat([x[..., H - pad:, :], x, x[..., :pad, :]], dim=2)
    x = torch.cat([x[..., W - pad:], x, x[..., :pad]], dim=3)
    x = torch.nn.functional.conv2d(x, filt.repeat(P_, 1, 1, 1), groups=P_)
    x = torch.relu(bn(x, (0, 2, 3), w1.view(1, -1, 1, 1), b1.view(1, -1, 1, 1)))
    x = x * torch.from_numpy(n1).double().view(B, P_ * F_, 1, 1)
    x = (x.reshape(B, -1) @ fw.t() + fb) * torch.from_numpy(n2).double()
    return torch.relu(bn(x, (0,), w2, b2)), P


@pytest.mark.parametrize("geom,B,G", [((2, 3, 3, 4, 3), 4, 2), ((3, 5, 5, 6, 4), 3, 1)])
def test_oracle_backward_matches_fp64_autograd(geom, B, G):
    """random tables, permutations and noise, repeated ids, G groups of B rows with their own statistics"""
    rng = np.random.RandomState(sum(geom) + B)
    N, R, Q = 9, 4, G * B
    P, F, ks, rh, rw = geom
    k = rh * rw
    st = itu.random_state(N, R, geom, seed=sum(geom))
    sd = {key: v for key, v in st.items()}
    e, r = rng.randint(N, size=Q), rng.randint(R, size=Q)
    e[1], r[2] = e[0], r[0]
    n0 = ((rng.rand(Q, P * 2 * k) > 0.3) / np.float32(0.7)).astype(np.float32)
    n1 = ((rng.rand(Q, P * F) > 0.2) / np.float32(0.8)).astype(np.float32)
    n2 = ((rng.rand(Q, k) > 0.3) / np.float32(0.7)).astype(np.float32)
    gx = rng.randn(Q, k)
    got, x64 = itu.oracle_bwd64(sd, e, r, B, gx, n0, n1, n2)
    want = [np.zeros(np.shape(sd[key])) for key in itu.PARAMS]
    for g0 in range(0, Q, B):
        s = slice(g0, g0 + B)
        x, Pt = _torch64(sd, e[s], r[s], n0[s], n1[s], n2[s])
        assert np.abs(x.detach().numpy() - x64[s]).max() <= 1e-9 * (1 + np.abs(x64).max())
        (x * torch.from_numpy(gx[s])).sum().backward()
        for i, p in enumerate(Pt):
            want[i] += p.grad.numpy()
    for key, a, b in zip(itu.PARAMS, got, want):
        assert np.abs(a - b).max() <= 1e-8 * (1 + np.abs(b).max()), key
    # the fp32 forward restates the same function
    x32 = itu.oracle_fwd(sd, e, r, B, n0, n1, n2)
    assert np.abs(x32 - x64).max() <= 1e-5 * (1 + np.abs(x64).max())
