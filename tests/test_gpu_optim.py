"""-m gpu tests of the optimizer kernels (kge_train.cu): the dense step kge_optim_apply_dense (SGD, Adagrad, Adam)
and the sparse step kge_optim_apply_rows (SGD, Adagrad), against oracle/ref_port.py's fp64 restatement of the
torch.optim update (pinned on the CPU by test_oracle_golden.py::test_ref_port_optimizer_steps_match_torch_optim)
and against torch.optim itself on the device.

Bounds, in units in the last place (ulp) of the float32 result:
  SGD       w' = w - lr g                        <= 1 ulp(w')                      (one fused rounding)
  Adagrad   s' = s + g g                         <= 1 ulp(s')
            w' = w - lr (g / (sqrt(s') + eps))   <= 1 ulp(w') + 2 ulp(lr g / (sqrt(s') + eps))
  Adam      m' = m + (g - m)(1 - b1)             <= 2 ulp of the largest of |m'|, |m|, |(1 - b1) g|
            v' = b2 v + (1 - b2) g g             <= 2 ulp(v')
            w' = w - step_size m' / denom        <= 1 ulp(w') + 4 ulp(update) + step_size |m'_kernel - m'| / denom
The Adagrad update rounds four times (sqrt, add, divide, multiply) and carries the rounding of s', hence 2 ulp;
Adam's weight bound carries the kernel's own error in m' (large only where m' cancels)."""
import numpy as np
import pytest
import torch

import gpu_util as gpu

pytestmark = pytest.mark.gpu

f32 = lambda x: float(np.float32(x))
LR = f32(0.05)
BETAS = (f32(0.9), f32(0.999))
EPS = {0: f32(1e-10), 1: f32(1e-10), 2: f32(1e-8)}
NAMES = {0: "sgd", 1: "adagrad", 2: "adam"}


def _L():
    from pykg2vec_b200 import _lib
    return _lib


def _ulp(x):
    return np.spacing(np.abs(np.asarray(x, dtype=np.float32))).astype(np.float64)


def _np(t):
    return t.detach().cpu().numpy().astype(np.float64) if torch.is_tensor(t) else np.asarray(t, np.float64)


def _within(got, want, bound, what):
    err = np.abs(_np(got) - _np(want))
    ratio = err / bound
    worst = int(np.argmax(ratio))
    assert ratio[worst] <= 1.0, "%s: element %d off by %.3g (bound %.3g)" % (what, worst, err[worst], bound[worst])
    return float(ratio[worst])


def _grad(rng, n):
    """magnitudes 1e-8 .. 10 with random signs, a quarter of the float4 chunks entirely zero (SGD / Adagrad skip
    those) and further single zeros (chunks that are only partly zero)."""
    g = rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 1, n)
    g[np.repeat(rng.rand((n + 3) // 4) < 0.25, 4)[:n]] = 0.0
    g[rng.rand(n) < 0.15] = 0.0
    return g.astype(np.float32)


def check_step(opt, w0, g, s10, s20, step, w1, s11, s21, lr=LR, eps=None, betas=BETAS):
    """One kernel step (w0, s10, s20 -> w1, s11, s21, all float32) against ref_port's fp64 step from the same
    float32 state.  Returns the worst error of each quantity as a fraction of its bound."""
    from oracle import ref_port
    eps = EPS[opt] if eps is None else eps
    w0, g, w1 = _np(w0), _np(g), _np(w1)
    worst = {}
    if opt == 0:
        want = ref_port.sgd_step(w0, g, lr).numpy()
        worst["w"] = _within(w1, want, _ulp(want), "sgd w")
    elif opt == 1:
        want, s = (x.numpy() for x in ref_port.adagrad_step(w0, g, _np(s10), lr, eps))
        worst["s"] = _within(s11, s, _ulp(s), "adagrad state_sum")
        worst["w"] = _within(w1, want, _ulp(want) + 2 * _ulp(want - w0), "adagrad w")
    else:
        m0 = _np(s10)
        want, m, v = (x.numpy() for x in ref_port.adam_step(w0, g, m0, _np(s20), step, lr, betas[0], betas[1], eps))
        worst["m"] = _within(s11, m, 2 * _ulp(np.maximum(np.maximum(np.abs(m), np.abs(m0)),
                                                        np.abs((1.0 - betas[0]) * g))), "adam exp_avg")
        worst["v"] = _within(s21, v, 2 * _ulp(v), "adam exp_avg_sq")
        step_size = lr / (1.0 - betas[0] ** step)
        denom = np.sqrt(v) / np.sqrt(1.0 - betas[1] ** step) + eps
        carried = step_size * np.abs(_np(s11) - m) / denom
        worst["w"] = _within(w1, want, _ulp(want) + 4 * _ulp(want - w0) + carried, "adam w")
    if opt != 2:   # SGD / Adagrad: elements without gradient keep their bits
        assert np.array_equal(gpu.bits(w1[g == 0]), gpu.bits(w0[g == 0]))
    return worst


def _big_n():
    # above three full sweeps of the kernel's grid cap (sm_count * 8 blocks of 256 threads, 4 floats each),
    # so the grid-stride loop runs, plus a 3-element scalar tail
    return 3 * torch.cuda.get_device_properties(0).multi_processor_count * 8 * 256 * 4 + 3


@pytest.mark.parametrize("opt", [0, 1, 2], ids=lambda o: NAMES[o])
@pytest.mark.parametrize("n", [1, 2, 3, 4, 5, 7, 1023, 4097, "big"])
def test_dense_apply_vs_fp64(opt, n):
    """kge_optim_apply_dense, three steps from the kernel's own state, each against the fp64 step; the gradient
    buffer is left zero-filled; under Adam elements without gradient still move."""
    L = _L()
    n = _big_n() if n == "big" else n
    rng = np.random.RandomState(n % 1000 + 10 * opt)
    w = torch.from_numpy((rng.standard_normal(n) * 0.5).astype(np.float32)).cuda()
    s1 = torch.from_numpy((rng.rand(n) * 0.1).astype(np.float32)).cuda() if opt == 1 else torch.zeros_like(w)
    s2 = torch.zeros_like(w)
    gbuf = torch.zeros_like(w)
    worst = {}
    for step in (1, 2, 3):
        g = _grad(rng, n)
        gbuf.copy_(torch.from_numpy(g))
        before = [x.cpu().numpy() for x in (w, s1, s2)]
        L.optim_apply_dense(w, gbuf, opt, LR, s1 if opt else None, s2 if opt == 2 else None, betas=BETAS, step=step)
        assert int(torch.count_nonzero(gbuf)) == 0, "gradient buffer must be left zero-filled"
        after = [x.cpu().numpy() for x in (w, s1, s2)]
        for k, v in check_step(opt, before[0], g, before[1], before[2], step, *after).items():
            worst[k] = max(worst.get(k, 0.0), v)
        if opt == 2 and step > 1:
            still = (g == 0) & (before[1] != 0)
            assert not still.any() or np.any(after[0][still] != before[0][still]), "Adam moves zero-gradient elements"
    print("dense %s n=%d worst error / bound: %s" % (NAMES[opt], n, {k: round(v, 3) for k, v in worst.items()}))


@pytest.mark.parametrize("foreach", [False, None], ids=["foreach_false", "foreach_default"])
@pytest.mark.parametrize("opt", [0, 1, 2], ids=lambda o: NAMES[o])
def test_dense_apply_tracks_torch_optim(opt, foreach):
    """20 steps of kge_optim_apply_dense == 20 steps of torch.optim.{SGD,Adagrad,Adam} on the same float32 tensor
    and the same gradients, on the device.  The two differ in rounding only (torch's float32 complement 1 - beta
    is rounded from a double, the kernel's is exact; fused multiply-adds differ), which accumulates over the
    steps: bounded by 5e-5 lr.  Measured on an H100 80GB HBM3 (400 W limit): SGD bit-identical, Adagrad 4.8e-6 lr,
    Adam 9.5e-6 lr, with and without foreach."""
    L = _L()
    n = 200003
    rng = np.random.RandomState(40 + opt)
    w0 = (rng.standard_normal(n) * 0.5).astype(np.float32)
    p = torch.from_numpy(w0.copy()).cuda().requires_grad_()
    kw = {} if foreach is None else {"foreach": foreach}
    topt = [torch.optim.SGD([p], lr=LR, **kw), torch.optim.Adagrad([p], lr=LR, **kw),
            torch.optim.Adam([p], lr=LR, **kw)][opt]
    w = torch.from_numpy(w0.copy()).cuda()
    s1, s2, gbuf = torch.zeros_like(w), torch.zeros_like(w), torch.zeros_like(w)
    for step in range(1, 21):
        g = torch.from_numpy(_grad(rng, n)).cuda()
        p.grad = g.clone()
        topt.step()
        gbuf.copy_(g)
        L.optim_apply_dense(w, gbuf, opt, LR, s1 if opt else None, s2 if opt == 2 else None, step=step)
    worst = float((w - p.detach()).abs().max()) / LR
    print("%s foreach=%s: max |w - torch| after 20 steps = %.3g lr" % (NAMES[opt], foreach, worst))
    assert worst <= 5e-5, worst


# every model the fused trainer steps; widths that are not multiples of 4 take the kernel's scalar path
SPARSE_MODELS = [("transe", 37, None), ("transh", 48, None), ("transd", 40, None), ("transr", 25, 13),
                 ("transm", 36, None), ("rotate", 64, None), ("rescal", 12, None), ("hole", 30, None),
                 ("kg2e", 40, None), ("distmult", 50, None), ("cp", 36, None), ("complex", 32, None),
                 ("simple", 48, None), ("analogy", 50, None), ("quate", 20, None), ("octonione", 12, None)]
ENTITY_KINDS = ("e", "e+", "e2")


@pytest.mark.parametrize("opt", [0, 1], ids=lambda o: NAMES[o])
@pytest.mark.parametrize("spec", SPARSE_MODELS, ids=lambda s: "%s-d%d" % (s[0], s[1]))
def test_sparse_apply_equals_dense_apply_and_fp64(spec, opt):
    """kge_optim_apply_rows on a gradient scratch filled by the model's own score_bwd over a batch with duplicate
    ids (ids that are head and tail, positive and negative): every table is bit-equal to kge_optim_apply_dense run
    on a copy of the same scratch, and within the fp64 bounds; rows the batch does not touch keep their bits; the
    scratch is zero afterwards."""
    L = _L()
    name, d, dr = spec
    N, R, B = 60, 5, 200
    om, tabs = gpu.synthetic_case(name, N, R, d, seed=17, dr=dr, scale=0.4)
    desc = gpu.desc_from_oracle_model(om)
    kinds = gpu.NUM_TABLE_SPECS[name]
    rng = np.random.RandomState(9)
    pos = [rng.randint(N, size=B), rng.randint(R, size=B), rng.randint(N, size=B)]
    pos[2][:20] = pos[0][:20]                                   # head == tail
    neg = [x.copy() for x in pos]
    neg[2][20:] = rng.randint(N, size=B - 20)                   # negatives share ids with the positives
    neg[0][::3] = pos[2][::3]                                   # a positive's tail as a negative's head
    pos[0][0], neg[2][0] = N - 1, 0                             # the first and the last entity row
    trained = [k != 2 if name == "transm" else True for k in range(len(tabs))]   # TransM's theta is not trained
    scratch = [torch.zeros_like(t) if trained[k] else None for k, t in enumerate(desc.tables)]
    ids = [[torch.from_numpy(x).cuda() for x in s] for s in (pos, neg)]
    for s, sign in zip(ids, (1.0, -1.0)):
        up = torch.from_numpy((sign * (0.5 + rng.rand(B))).astype(np.float32)).cuda()
        L.score_bwd(desc, *s, up, [x if x is not None else torch.zeros_like(desc.tables[k])
                                   for k, x in enumerate(scratch)])
    state = [torch.from_numpy((rng.rand(*t.shape) * 0.1).astype(np.float32)).cuda() for t in tabs] if opt else None
    w0 = [t.clone() for t in desc.tables]
    g0 = [x.clone() if x is not None else None for x in scratch]
    s0 = [x.clone() for x in state] if opt else None
    assert any(float(x.abs().max()) > 0 for x in g0 if x is not None)
    for s in ids:                                               # as Trainer._apply does: one call per id set
        L.optim_apply_rows(desc, scratch, state, opt, *s, LR)
    assert all(int(torch.count_nonzero(x)) == 0 for x in scratch if x is not None), "scratch must be left zero"
    used = {"e": np.unique(np.concatenate([pos[0], pos[2], neg[0], neg[2]])), "r": np.unique(np.concatenate([pos[1], neg[1]]))}
    for k, t in enumerate(desc.tables):
        if not trained[k]:
            assert torch.equal(t, w0[k])
            continue
        wd, gd = w0[k].clone(), g0[k].clone()
        sd = s0[k].clone() if opt else None
        L.optim_apply_dense(wd, gd, opt, LR, sd)
        assert np.array_equal(gpu.bits(t.cpu().numpy()), gpu.bits(wd.cpu().numpy())), \
            "%s table %d: sparse != dense apply (%d elements differ)" % (name, k, int((t != wd).sum()))
        if opt:
            assert torch.equal(state[k], sd), "%s state %d: sparse != dense apply" % (name, k)
        check_step(opt, w0[k].cpu().numpy().ravel(), g0[k].cpu().numpy().ravel(),
                   s0[k].cpu().numpy().ravel() if opt else None, None, 1, t.cpu().numpy().ravel(),
                   state[k].cpu().numpy().ravel() if opt else None, None)
        if t.dim() == 2:   # rows of this table's kind that no id of the batch names keep their bits
            rows = used["e" if kinds[k] in ENTITY_KINDS else "r"]
            untouched = np.setdiff1d(np.arange(t.shape[0]), rows)
            assert len(untouched) > 0 or t.shape[0] <= len(rows)
            assert np.array_equal(gpu.bits(t.cpu().numpy()[untouched]), gpu.bits(w0[k].cpu().numpy()[untouched]))


def test_optimizer_argument_errors_write_nothing():
    L = _L()
    n = 1027
    w = torch.randn(n + 1, device="cuda")
    g = torch.randn(n + 1, device="cuda")
    s1, s2 = torch.zeros_like(w), torch.zeros_like(w)
    keep = [x.clone() for x in (w, g, s1, s2)]
    with pytest.raises(L.KgeError, match="aligned"):            # a view one float into its storage
        L.optim_apply_dense(w[1:], g[1:], L.OPT_SGD, LR)
    with pytest.raises(L.KgeError):
        L.optim_apply_dense(w[1:], g[1:], L.OPT_ADAM, LR, s1[1:], s2[1:], step=1)
    with pytest.raises(L.KgeError):                             # Adam's bias correction needs step >= 1
        L.optim_apply_dense(w, g, L.OPT_ADAM, LR, s1, s2, step=0)
    with pytest.raises(L.KgeError):                             # Adagrad without its state table
        L.optim_apply_dense(w, g, L.OPT_ADAGRAD, LR, None)
    om, tabs = gpu.synthetic_case("transe", 50, 4, 32, seed=1)
    desc = gpu.desc_from_oracle_model(om)
    scratch = [torch.ones_like(t) for t in desc.tables]
    h = torch.arange(8, device="cuda")
    with pytest.raises(L.KgeError, match="state"):
        L.optim_apply_rows(desc, scratch, None, L.OPT_ADAGRAD, h, h % 4, h, LR)
    torch.cuda.synchronize()
    for a, b in zip((w, g, s1, s2), keep):
        assert torch.equal(a, b), "a rejected call wrote to its arguments"
    assert all(torch.equal(t, torch.from_numpy(x).cuda()) for t, x in zip(desc.tables, tabs))
    assert all(bool((s == 1).all()) for s in scratch)
