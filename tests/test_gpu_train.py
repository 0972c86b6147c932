"""-m gpu tests of the training-side kernels: backward vs the fp64 autograd oracle
(oracle/ref_port.py) and vs gradients produced by the reference itself (golden), losses,
regularisers, the model classes through autograd, and the fused sparse training steps vs
dense torch optimizers on the oracle formulas."""
import numpy as np
import pytest
import torch

import golden_util as gu
import gpu_util as gpu

pytestmark = pytest.mark.gpu
CASES = [n for n in gu.case_names() if "pretrained" not in n]
GRAD_TOL = 2e-4  # relative to the largest |gradient| of the table


def _L():
    from pykg2vec_b200 import _lib
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _check_grads(got, want, tol=GRAD_TOL, what=""):
    for k, (g, w) in enumerate(zip(got, want)):
        if w is None:
            continue
        w = np.asarray(w, dtype=np.float64)
        scale = max(np.abs(w).max(), 1e-12)
        err = np.abs(g.astype(np.float64) - w).max() / scale
        assert err < tol, "%s table %d: rel err %.3g" % (what, k, err)


@pytest.mark.parametrize("name", CASES)
def test_score_bwd_vs_reference_autograd(name):
    L = _L()
    g = gu.load(name)
    desc = gpu.desc_from_golden(g)
    grads = [torch.zeros_like(t) for t in desc.tables]
    L.score_bwd(desc, _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"]), _cuda(g["upstream"]), grads)
    want = [g.get("grad%d" % k) for k in range(len(grads))]   # (ConvKB: no reference gradient for the collapsed tables)
    _check_grads([x.cpu().numpy() for x in grads], want, what=name)


@pytest.mark.parametrize("spec", [
    ("transe", 300, 7, 200, None, False, 0.0), ("transe", 300, 7, 50, None, True, 0.0),
    ("transh", 300, 7, 100, None, True, 0.0), ("transd", 300, 7, 64, None, False, 0.0),
    ("transr", 120, 5, 40, 24, False, 0.0), ("transm", 300, 7, 36, None, False, 0.0),
    ("rotate", 300, 7, 100, None, False, 12.0), ("distmult", 300, 7, 200, None, False, 0.0),
    ("cp", 300, 7, 30, None, False, 0.0), ("complex", 300, 7, 200, None, False, 0.0),
    ("hole", 200, 5, 30, None, False, 0.0), ("hole", 200, 5, 52, None, False, 0.0),
    ("rescal", 150, 4, 24, None, False, 0.0), ("simple", 300, 7, 48, None, False, 0.0),
    ("simple_ignr", 300, 7, 50, None, False, 0.0), ("analogy", 300, 7, 48, None, False, 0.0),
    ("slm", 200, 5, 24, 16, False, 0.0), ("ntn", 120, 4, 16, 12, False, 0.0), ("sme", 150, 5, 24, None, False, 0.0),
    ("sme_bl", 150, 5, 20, None, False, 0.0), ("kg2e", 200, 5, 40, None, False, 0.0), ("quate", 200, 5, 24, None, False, 0.0), ("octonione", 150, 5, 12, None, False, 0.0),
    ("convkb", 200, 5, 50, None, False, 0.0), ("convkb", 150, 5, 37, None, False, 0.0),
], ids=lambda s: "%s-d%d" % (s[0], s[3]))
def test_score_bwd_vs_fp64_oracle(spec):
    """duplicates in the batch (few entities) exercise the atomic scatter."""
    from oracle import ref_port
    L = _L()
    name, N, R, d, dr, l1, margin = spec
    om, tabs = gpu.synthetic_case(name, N, R, d, seed=11, dr=dr, l1=l1, margin=margin, scale=0.3)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(1)
    n = 777
    h, r, t = rng.randint(N, size=n), rng.randint(R, size=n), rng.randint(N, size=n)
    up = rng.standard_normal(n).astype(np.float32)
    grads = [torch.zeros_like(x) for x in desc.tables]
    L.score_bwd(desc, _cuda(h), _cuda(r), _cuda(t), _cuda(up), grads)
    t64 = [torch.from_numpy(x.astype(np.float64)).requires_grad_(name != "transm" or i < 2)
           for i, x in enumerate(tabs)]
    s = ref_port.score(name, t64, torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t),
                       l1_flag=l1, margin=margin, embedding_range=((margin + 2.0) / d if name == "rotate" else None),
                       rel_dim=dr)
    (s * torch.from_numpy(up.astype(np.float64))).sum().backward()
    want = [x.grad.numpy() if x.grad is not None else None for x in t64]
    _check_grads([x.cpu().numpy() for x in grads], want, tol=5e-5, what=name)


def test_losses_vs_golden_and_oracle():
    import oracle
    L = _L()
    g = gu.load("losses")
    loss, gp, gn = L.loss_pairwise_hinge(_cuda(g["pos"]), _cuda(g["neg"]), float(g["margin"]))
    assert abs(loss.item() - g["hinge"]) <= 1e-5 * abs(g["hinge"])
    np.testing.assert_array_equal(gp.cpu().numpy(), g["hinge_gpos"])
    np.testing.assert_array_equal(gn.cpu().numpy(), g["hinge_gneg"])
    loss, gg = L.loss_pointwise_logistic(_cuda(g["preds"]), _cuda(g["target"]))
    assert abs(loss.item() - g["logistic"]) <= 1e-5 * abs(g["logistic"])
    np.testing.assert_allclose(gg.cpu().numpy(), g["logistic_g"], rtol=1e-4, atol=1e-8)
    for tag, alpha in (("a1", 1.0), ("a01", 0.1)):
        loss, gp, gn = L.loss_selfadv(_cuda(g["sa_pos"]), _cuda(g["sa_neg"]), int(g["sa_neg_rate"]), alpha)
        assert abs(loss.item() - g["sa_" + tag]) <= 2e-5 * abs(g["sa_" + tag])
        np.testing.assert_allclose(gp.cpu().numpy(), g["sa_%s_gpos" % tag], rtol=1e-4, atol=1e-8)
        np.testing.assert_allclose(gn.cpu().numpy(), g["sa_%s_gneg" % tag], rtol=1e-4, atol=1e-8)
    # larger, seeded: vs the C oracle
    rng = np.random.RandomState(3)
    pos = (rng.standard_normal(5000) * 2).astype(np.float32)
    neg = (rng.standard_normal(5000) * 2).astype(np.float32)
    want, _ = oracle.loss_pairwise_hinge(pos, neg, 1.5)
    got, _, _ = L.loss_pairwise_hinge(_cuda(pos), _cuda(neg), 1.5)
    assert abs(got.item() - want) <= 1e-5 * abs(want)
    neg2 = (rng.standard_normal(5000 * 16) * 3).astype(np.float32)
    want = oracle.loss_selfadv(pos, neg2, 16, 0.5)
    got, _, _ = L.loss_selfadv(_cuda(pos), _cuda(neg2), 16, 0.5)
    assert abs(got.item() - want) <= 2e-5 * abs(want)


@pytest.mark.parametrize("name", [n for n in CASES if n.split("_")[0] in ("distmult", "complex", "cp", "analogy", "quate", "octonione")])
def test_regulariser_vs_golden_and_autograd(name):
    from oracle import ref_port
    L = _L()
    g = gu.load(name)
    desc = gpu.desc_from_golden(g)
    h, r, t = _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])
    lm = float(g["kw_lmbda"])
    for code, key in ((0, "reg_f2"), (1, "reg_n3"), (2, "reg_absn3")):
        if key not in g:
            continue
        grads = [torch.zeros_like(x) for x in desc.tables]
        out = L.reg_fwd_bwd(desc, code, lm, h, r, t, grad_scale=1.0, grad_tables=grads)
        assert abs(out.item() - g[key]) <= 1e-4 * abs(g[key]) + 1e-9, (name, key)
        t64 = [torch.from_numpy(x.astype(np.float64)).requires_grad_() for x in gu.tables_of(g)]
        ref_port.reg(str(g["model"]), t64, torch.from_numpy(g["h"]), torch.from_numpy(g["r"]),
                     torch.from_numpy(g["t"]), lm, code).backward()
        _check_grads([x.cpu().numpy() for x in grads], [x.grad.numpy() for x in t64], tol=5e-5, what=name + key)


def _make_model(g, device="cuda"):
    """the pykg2vec_b200 model class for a golden case, loaded with the golden tables through
    the reference's state_dict keys."""
    import pykg2vec_b200
    kw = {k[3:]: (g[k].item() if g[k].ndim == 0 else g[k]) for k in g if k.startswith("kw_")}
    cls = pykg2vec_b200.import_model(str(g["model"]))
    if str(g["model"]) == "convkb":
        kw["device"] = device   # the reference's ConvKB takes the device of its (unregistered) conv_list
    m = cls(tot_entity=int(g["N"]), tot_relation=int(g["R"]), **kw)
    sd = {str(k) + ".weight": torch.from_numpy(g["table%d" % i]) for i, k in enumerate(g["table_keys"])}
    if str(g["model"]) == "convkb":
        raw = gu.raw_tables_of(g)
        sd["fc1.weight"], sd["fc1.bias"] = torch.from_numpy(raw[-2]), torch.from_numpy(raw[-1])
        with torch.no_grad():
            for i, conv in enumerate(m.conv_list):   # plain Python list: not part of state_dict
                conv.weight.copy_(torch.from_numpy(raw[2 + 2 * i]))
                conv.bias.copy_(torch.from_numpy(raw[3 + 2 * i]))
    missing = m.load_state_dict(sd, strict=False)  # (QuatE/OctonionE register tables forward() never reads)
    assert not missing.unexpected_keys
    return m.to(device)


@pytest.mark.parametrize("name", CASES)
def test_model_classes_forward_backward_like_reference(name):
    """Drop-in surface: state_dict keys load, forward() scores and .backward() dense grads
    match what the reference classes produced."""
    g = gu.load(name)
    if str(g["model"]) == "transm":
        pytest.skip("needs a knowledge graph")
    if str(g["model"]) == "rescal":
        pytest.skip("forward() re-normalises the stored (already normalised) tables: covered by test_rescal_model")
    m = _make_model(g)
    h, r, t = _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])
    s = m(h, r, t)
    ref = g["scores"]
    floor = 1e-2 * np.abs(ref).max()
    err = np.abs(s.detach().cpu().numpy().astype(np.float64) - ref) / np.maximum(np.abs(ref), floor)
    assert err.max() < 1e-4
    (s * _cuda(g["upstream"])).sum().backward()
    got = [getattr(m, str(k)).weight.grad.cpu().numpy() for k in g["table_keys"]]
    _check_grads(got, [g["grad%d" % i] for i in range(len(got))], what=name)
    if str(g["model"]) == "convkb":   # the Linear layer trains through the collapse
        raw_n = len(gu.raw_tables_of(g))
        _check_grads([m.fc1.weight.grad.cpu().numpy(), m.fc1.bias.grad.cpu().numpy()],
                     [g["rawgrad%d" % (raw_n - 2)], g["rawgrad%d" % (raw_n - 1)]], what=name + " fc1")
        assert "conv_list" not in "".join(m.state_dict().keys())
    embs = m.embed(h, r, t)
    assert all(e.shape[0] == h.numel() for e in embs)


def test_fused_hinge_sgd_matches_dense_sgd():
    """kge_train_pairwise_hinge_sgd == (oracle formulas + torch autograd + optim.SGD)."""
    from oracle import ref_port
    L = _L()
    for name, d, dr, l1 in (("transe", 200, None, False), ("transe", 50, None, True), ("transh", 48, None, False),
                            ("transd", 40, None, True), ("transr", 25, 13, False), ("transm", 36, None, False),
                            ("kg2e", 40, None, False), ("hole", 30, None, False)):
        N, R, B = 500, 9, 512
        om, tabs = gpu.synthetic_case(name, N, R, d, seed=21, dr=dr, l1=l1, scale=0.4)
        desc = gpu.desc_from_oracle_model(om)
        if name == "kg2e":   # variances in [1.05, 2.05]: three SGD steps keep them positive (the score takes log)
            for k in (1, 3):
                desc.tables[k].add_(1.0)
                tabs[k] = tabs[k] + np.float32(1.0)
        scratch = [torch.zeros_like(x) for x in desc.tables]
        # (TransM's per-relation theta is not a trained parameter)
        ref = [torch.from_numpy(x.astype(np.float64)).requires_grad_(name != "transm" or k < 2) for k, x in enumerate(tabs)]
        opt = torch.optim.SGD([x for x in ref if x.requires_grad], lr=0.05)
        rng = np.random.RandomState(4)
        for step in range(3):
            ids = [rng.randint(N if k % 3 != 1 else R, size=B) for k in range(6)]
            loss = L.train_pairwise_hinge_sgd(desc, scratch, *[_cuda(x) for x in ids], margin=0.7, lr=0.05)
            opt.zero_grad()
            tid = [torch.from_numpy(x) for x in ids]
            pos = ref_port.score(name, ref, tid[0], tid[1], tid[2], l1_flag=l1)
            neg = ref_port.score(name, ref, tid[3], tid[4], tid[5], l1_flag=l1)
            want = ref_port.pairwise_hinge(pos, neg, 0.7)
            want.backward()
            opt.step()
            assert abs(loss.item() - want.item()) <= 2e-4 * abs(want.item()), (name, step)
            for a, b in zip(desc.tables, ref):
                np.testing.assert_allclose(a.cpu().numpy(), b.detach().numpy(), rtol=0, atol=3e-5, err_msg=name)
            assert all(float(s.abs().max()) == 0.0 for s in scratch), "gradient scratch must be left zeroed"


@pytest.mark.parametrize("neg_rate,B", [(1, 70), (3, 129), (4, 64), (5, 33), (16, 64), (256, 40)])
def test_fused_selfadv_step_equals_the_five_launch_path(neg_rate, B):
    """kge_train_pairwise_selfadv (RotatE: forward + self-adversarial loss + backward in one kernel; a warp per
    positive up to neg_rate 4, a CTA per positive beyond) == kge_score_fwd x2 + kge_loss_selfadv + kge_score_bwd x2:
    the loss terms are the same bits (summed by unordered atomics -> compared to fp32 rounding), the gradients
    equal up to the order of the float atomics."""
    L = _L()
    N, R, d = 700, 9, 100
    om, tabs = gpu.synthetic_case("rotate", N, R, d, seed=31)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(neg_rate)
    ids = [_cuda(rng.randint(N if k % 3 != 1 else R, size=B if k < 3 else B * neg_rate)) for k in range(6)]
    g_fused = [torch.zeros_like(x) for x in desc.tables]
    loss_fused = L.train_pairwise_selfadv(desc, g_fused, *ids, neg_rate=neg_rate, alpha=0.5)
    pos, neg = L.score_fwd(desc, *ids[:3]), L.score_fwd(desc, *ids[3:])
    loss, gp, gn = L.loss_selfadv(pos, neg, neg_rate, 0.5)
    g_ref = [torch.zeros_like(x) for x in desc.tables]
    L.score_bwd(desc, *ids[:3], gp, g_ref)
    L.score_bwd(desc, *ids[3:], gn, g_ref)
    assert abs(loss_fused.item() - loss.item()) <= 2e-6 * abs(loss.item())
    _check_grads([g.cpu().numpy() for g in g_fused], [g.cpu().numpy() for g in g_ref], tol=2e-5, what="selfadv fused")
    with pytest.raises(L.KgeNotSupported):   # other models do not train with this loss
        om2, _ = gpu.synthetic_case("transe", N, R, d, seed=1)
        d2 = gpu.desc_from_oracle_model(om2)
        L.train_pairwise_selfadv(d2, [torch.zeros_like(x) for x in d2.tables], *ids, neg_rate=neg_rate, alpha=0.5)


# table scale per pointwise model: at least 10% of the batch on each side of |y s| = 20, the softplus threshold
POINTWISE_SCALE = {"distmult": 2.0, "complex": 1.5, "cp": 2.0, "simple": 1.5, "simple_ignr": 1.5, "analogy": 1.5,
                   "quate": 2.0, "octonione": 2.0}


@pytest.mark.parametrize("name", sorted(POINTWISE_SCALE))
def test_fused_pointwise_step_vs_fp64(name):
    """kge_train_pointwise_logistic (forward + Criterion.pointwise_logistic + backward in one kernel) == ref_port's
    score and pointwise_logistic in float64 autograd, on both branches of F.softplus's threshold."""
    from oracle import ref_port
    L = _L()
    N, R, d, B = 40, 5, (16 if name == "quate" else 8 if name == "octonione" else 32), 512
    om, tabs = gpu.synthetic_case(name, N, R, d, seed=7, scale=POINTWISE_SCALE[name])
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(3)
    h, r, t = rng.randint(N, size=B), rng.randint(R, size=B), rng.randint(N, size=B)
    y = np.where(rng.rand(B) < 0.5, 1, -1).astype(np.int64)
    scratch = [torch.zeros_like(x) for x in desc.tables]
    loss = L.train_pointwise_logistic(desc, scratch, _cuda(h), _cuda(r), _cuda(t), _cuda(y))
    t64 = [torch.from_numpy(x.astype(np.float64)).requires_grad_() for x in tabs]
    s = ref_port.score(name, t64, torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t))
    x = (torch.from_numpy(y).double() * s).detach().numpy()
    if name.startswith("simple"):
        # SimplE clamps its score to [-20, 20] (pointwise.py:514-526): |y s| never exceeds the threshold, and the
        # clamped triples (exactly on it, zero gradient) are the other side
        assert (np.abs(x) >= 20).mean() >= 0.1 and (np.abs(x) < 20).mean() >= 0.1, (np.abs(x) >= 20).mean()
    else:
        assert (x > 20).mean() >= 0.1 and (x <= 20).mean() >= 0.1, (x > 20).mean()
    want = ref_port.pointwise_logistic(s, torch.from_numpy(y).double())
    want.backward()
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item()), (loss.item(), want.item())
    _check_grads([g.cpu().numpy() for g in scratch], [x.grad.numpy() for x in t64], tol=5e-5, what=name)


def _distmult_exact_scores(a):
    """DistMult rows whose scores are exact in float32: h_i = (a_i, 0, 0, 0), r = t = (1, 0, 0, 0) -> s_i = -a_i,
    and d s_i / d h_i = (-1, 0, 0, 0): the gradient row of triple i is exactly -d loss / d s_i (one triple per row)."""
    n = len(a)
    ent = np.zeros((n + 1, 4), np.float32)
    ent[:n, 0], ent[n, 0] = a, 1.0
    rel = np.zeros((1, 4), np.float32)
    rel[0, 0] = 1.0
    import oracle
    desc = gpu.desc_from_oracle_model(oracle.Model("distmult", [ent, rel], 4))
    return desc, np.arange(n), np.zeros(n, np.int64), np.full(n, n)


def _logistic_edge_inputs():
    """y s on both sides of 20 (and the neighbouring floats), and in (15, 16.5) where sigmoid(y s) is still
    several ulp below 1 in float32: a kernel that switched to the y s branch too early is visible there."""
    up = np.float32(20.0)
    x = np.array([np.nextafter(up, np.float32(0)), up, np.nextafter(up, np.float32(30)), 15.0, 15.25, 15.5, 16.0,
                  16.25, 14.0, 10.0, 0.5, 0.0, -3.0, -15.0, -20.0, 20.5, 25.0, 40.0], np.float32)
    y = np.where(np.arange(len(x)) % 2 == 0, 1, -1).astype(np.int64)
    return x, y


def test_fused_logistic_threshold_vs_fp64():
    """train_logistic_kernel at y s = 20, its float neighbours, and 15 .. 16.5: per-triple gradients against
    float64 F.softplus' derivative (torch's threshold rule: y s > 20 -> gradient exactly 1).  For y s >= 14,
    sigmoid(y s) = 1 / (1 + exp(-y s)) rounds twice near 1 (<= 1.5 ulp); below, expf's own error (2 ulp) enters."""
    from oracle import ref_port
    L = _L()
    x, y = _logistic_edge_inputs()
    n = 32   # (a power of two: 1/n is exact)
    x = np.resize(x, n)
    y = np.resize(y, n)
    a = (-x * y).astype(np.float32)          # s = -a, so y s = x exactly
    desc, h, r, t = _distmult_exact_scores(a)
    scratch = [torch.zeros_like(w) for w in desc.tables]
    loss = L.train_pointwise_logistic(desc, scratch, _cuda(h), _cuda(r), _cuda(t), _cuda(y))
    s = torch.from_numpy(-a.astype(np.float64)).requires_grad_()
    want = ref_port.pointwise_logistic(s, torch.from_numpy(y).double())
    want.backward()
    got = -scratch[0][:n, 0].cpu().numpy().astype(np.float64)
    ref = s.grad.numpy()
    err = np.abs(got - ref) / np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)
    bound = np.where(x >= 14, 1.5, 4.0)
    worst = int(np.argmax(err / bound))
    assert err[worst] <= bound[worst], (x[worst], got[worst], ref[worst], err[worst])
    assert abs(loss.item() - want.item()) <= 2e-6 * abs(want.item())


@pytest.mark.parametrize("neg_rate", [1, 5, 33, 256])
@pytest.mark.parametrize("alpha", [0.0, 1.0, 30.0])
def test_fused_selfadv_step_vs_fp64(neg_rate, alpha):
    """kge_train_pairwise_selfadv == ref_port.score + ref_port.selfadv in float64 autograd, with scores in about
    [-3, 3]: at alpha 30, alpha |s| reaches ~100, where the softmax overflows float32 without the max shift.
    The softmax weights carry alpha times the float32 score error (~1e-6), hence the alpha term in the tolerance."""
    from oracle import ref_port
    L = _L()
    N, R, d, B, margin = 80, 6, 16, 24, 4.0
    om, tabs = gpu.synthetic_case("rotate", N, R, d, seed=31, margin=margin, scale=0.25)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(neg_rate)
    ids = [rng.randint(N if k % 3 != 1 else R, size=B if k < 3 else B * neg_rate) for k in range(6)]
    scratch = [torch.zeros_like(x) for x in desc.tables]
    loss = L.train_pairwise_selfadv(desc, scratch, *[_cuda(x) for x in ids], neg_rate=neg_rate, alpha=alpha)
    t64 = [torch.from_numpy(x.astype(np.float64)).requires_grad_() for x in tabs]
    sc = lambda a, b, c: ref_port.score("rotate", t64, *(torch.from_numpy(v) for v in (a, b, c)), margin=margin,
                                        embedding_range=(margin + 2.0) / d)
    pos, neg = sc(*ids[:3]), sc(*ids[3:])
    if alpha == 30.0:
        assert float((alpha * neg.abs()).max()) > 80.0
    want = ref_port.selfadv(pos, neg, neg_rate, alpha)
    want.backward()
    assert np.isfinite(loss.item())
    assert abs(loss.item() - want.item()) <= (1e-5 + alpha * 1e-6) * abs(want.item()), (loss.item(), want.item())
    _check_grads([g.cpu().numpy() for g in scratch], [x.grad.numpy() for x in t64], tol=5e-5 + alpha * 2e-6,
                 what="selfadv fused")


@pytest.mark.parametrize("n", [1, 1023, 1024, 1025, 100003])
def test_loss_kernels_vs_fp64(n):
    """kge_loss_pairwise_hinge / kge_loss_pointwise_logistic (one 1024-thread CTA looping over n) == ref_port's
    losses in float64 autograd, below, at and above one element per thread."""
    from oracle import ref_port
    L = _L()
    rng = np.random.RandomState(n)
    pos = (rng.standard_normal(n) * 2).astype(np.float32)
    neg = (rng.standard_normal(n) * 2).astype(np.float32)
    margin = 0.75
    p64 = torch.from_numpy(pos.astype(np.float64)).requires_grad_()
    n64 = torch.from_numpy(neg.astype(np.float64)).requires_grad_()
    v = np.float32(pos + np.float32(margin)) - neg
    assert not (v == 0).any()   # exact ties are pinned on their own (test_hinge_exact_tie_has_zero_gradient)
    want = ref_port.pairwise_hinge(p64, n64, margin)
    want.backward()
    loss, gp, gn = L.loss_pairwise_hinge(_cuda(pos), _cuda(neg), margin)
    assert abs(loss.item() - want.item()) <= 1e-5 * max(abs(want.item()), 1e-30), (loss.item(), want.item())
    np.testing.assert_array_equal(gp.cpu().numpy(), p64.grad.numpy())
    np.testing.assert_array_equal(gn.cpu().numpy(), n64.grad.numpy())
    preds = (rng.standard_normal(n) * 12).astype(np.float32)     # a share of |y s| beyond the threshold 20
    y = np.where(rng.rand(n) < 0.5, 1.0, -1.0).astype(np.float32)
    if n >= 20:
        x, yy = _logistic_edge_inputs()
        preds[:len(x)], y[:len(x)] = x * yy, yy                 # y s on the threshold and its neighbours
    s64 = torch.from_numpy(preds.astype(np.float64)).requires_grad_()
    want = ref_port.pointwise_logistic(s64, torch.from_numpy(y.astype(np.float64)))
    want.backward()
    loss, g = L.loss_pointwise_logistic(_cuda(preds), _cuda(y))
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item()), (loss.item(), want.item())
    ref = s64.grad.numpy()
    np.testing.assert_allclose(g.cpu().numpy(), ref, rtol=2e-6, atol=1e-6 * np.abs(ref).max())


@pytest.mark.parametrize("neg_rate", [1, 5, 33, 256])
def test_loss_selfadv_vs_fp64_at_extremes(neg_rate):
    """kge_loss_selfadv (a warp per positive, lane-strided over the negatives) == ref_port.selfadv in float64 at
    alpha |s| up to ~100 on either sign, where exp without the max shift overflows or underflows float32."""
    from oracle import ref_port
    L = _L()
    B = 37
    rng = np.random.RandomState(50 + neg_rate)
    pos = (rng.standard_normal(B) * 2).astype(np.float32)
    neg = rng.uniform(-3.3, 3.3, B * neg_rate).astype(np.float32)
    for alpha in (0.0, 1.0, 30.0):
        p64 = torch.from_numpy(pos.astype(np.float64)).requires_grad_()
        n64 = torch.from_numpy(neg.astype(np.float64)).requires_grad_()
        want = ref_port.selfadv(p64, n64, neg_rate, alpha)
        want.backward()
        loss, gp, gn = L.loss_selfadv(_cuda(pos), _cuda(neg), neg_rate, alpha)
        # (the float32 exponent -alpha s - max carries ~alpha * 4e-7 of rounding, hence the alpha terms)
        assert abs(loss.item() - want.item()) <= (1e-5 + alpha * 1e-6) * abs(want.item()), (alpha, loss.item(), want.item())
        np.testing.assert_allclose(gp.cpu().numpy(), p64.grad.numpy(), rtol=1e-5, atol=0)
        ref = n64.grad.numpy()
        np.testing.assert_allclose(gn.cpu().numpy(), ref, rtol=1e-5 + alpha * 1e-6, atol=1e-6 * np.abs(ref).max(),
                                   err_msg=str(alpha))


def test_hinge_exact_tie_has_zero_gradient():
    """pos + margin == neg bit for bit: the hinge term is 0 and the kernels give it ZERO gradient (`v > 0`), in
    the loss kernel and in the fused hinge + SGD step (the tables do not move).  torch.max(v, zeros), which
    ref_port.pairwise_hinge restates, splits the gradient of a tie (0.5 to each argument) in current torch; the
    reference pins torch < 1.7, whose tie rule is not checked here.  The fp64 comparisons keep ties out."""
    L = _L()
    pos = np.array([0.25, -1.0, 3.5, 0.5], np.float32)
    neg = np.array([1.0, -0.25, 4.25, 0.0], np.float32)   # pos + 0.75 == neg exactly, except the last (active)
    loss, gp, gn = L.loss_pairwise_hinge(_cuda(pos), _cuda(neg), 0.75)
    assert loss.item() == 1.25
    np.testing.assert_array_equal(gp.cpu().numpy(), [0, 0, 0, 1])
    np.testing.assert_array_equal(gn.cpu().numpy(), [0, 0, 0, -1])
    # the fused step: every negative is its positive, so with margin 0 every pair is an exact tie
    om, tabs = gpu.synthetic_case("transe", 20, 3, 16, seed=2)
    desc = gpu.desc_from_oracle_model(om)
    scratch = [torch.zeros_like(x) for x in desc.tables]
    ids = [_cuda(np.array([3, 5])), _cuda(np.array([1, 2])), _cuda(np.array([7, 9]))]
    loss = L.train_pairwise_hinge_sgd(desc, scratch, *ids, *ids, margin=0.0, lr=0.5)
    assert loss.item() == 0.0
    for w, w0 in zip(desc.tables, tabs):
        assert np.array_equal(gpu.bits(w.cpu().numpy()), gpu.bits(w0))


def _trainer_for(model_name, kg, **cfgkw):
    import pykg2vec_b200
    from pykg2vec_b200.synthetic import SyntheticConfig
    from pykg2vec_b200.trainer import Trainer
    cfg = SyntheticConfig(kg, **cfgkw)
    torch.manual_seed(0)
    model = pykg2vec_b200.import_model(model_name)(**cfg.__dict__)
    tr = Trainer(model, cfg)
    tr.build_model()
    return tr


def _trainer_rows():
    rows = [
        ("transe", "sgd"), ("transe", "adagrad"), ("distmult", "sgd"), ("complex", "adagrad"), ("rotate", "adagrad"),
        # every pointwise model with its own get_reg default (ADVICE r1: SimplE's id-tensor regulariser, QuatE /
        # OctonionE |x|^3, CP signed x^3, ComplexN3 |x|^3), and Rescal whose forward() normalises in place
        ("cp", "sgd"), ("complexn3", "sgd"), ("analogy", "adagrad"), ("simple", "sgd"), ("simple_ignr", "adagrad"),
        ("quate", "sgd"), ("octonione", "adagrad"), ("rescal", "sgd"), ("rescal", "adagrad"), ("hole", "sgd"),
        ("transh", "sgd"), ("transd", "adagrad"), ("kg2e", "sgd"), ("transr", "adagrad"), ("transm", "sgd"),
        # Adam, the CLI default: kge_optim_apply_dense over every table
        ("transe", "adam"), ("distmult", "adam"), ("complex", "adam"), ("quate", "adam"), ("analogy", "adam"),
        ("transr", "adam"), ("kg2e", "adam"), ("rotate", "adam")]
    extra = [("rotate", "adam", {"neg_rate": 16}),                            # the CTA-team self-adversarial step
             ("transe", "adagrad", {"hidden_size": 37}),                      # scalar path of the sparse Adagrad
             ("transr", "adagrad", {"ent_hidden_size": 25, "rel_hidden_size": 13})]
    return [pytest.param(m, o, {}, id="%s-%s" % (m, o)) for m, o in rows] + \
        [pytest.param(m, o, kw, id="-".join([m, o] + ["%s%d" % kv for kv in kw.items()])) for m, o, kw in extra]


@pytest.mark.parametrize("model_name,opt,override", _trainer_rows())
def test_trainer_fused_equals_autograd_mode(model_name, opt, override):
    """Trainer.train_batch in fused mode follows the same weight trajectory as the autograd
    mode (reference step order) with the dense torch optimizer."""
    from pykg2vec_b200.synthetic import SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(400, 6, 2000, 50, 50, seed=1)
    kw = dict(optimizer=opt, learning_rate=0.05, hidden_size=32 if model_name == "rescal" else 64,
              ent_hidden_size=64, rel_hidden_size=64, margin=1.0 if model_name != "rotate" else 6.0,
              l1_flag=False, lmbda=0.01, neg_rate=4 if model_name == "rotate" else 1, alpha=0.5,
              cmax=0.5, cmin=-0.5, batch_size=256)
    kw.update(override)
    a = _trainer_for(model_name, kg, fused_step=True, **kw)
    b = _trainer_for(model_name, kg, fused_step=False, **kw)
    b.model.load_state_dict(a.model.state_dict())
    assert a._fused and not b._fused
    rng = np.random.RandomState(2)
    B, steps, atol = 256, 3, 2e-5
    for step in range(steps):
        if a.model.training_strategy.name == "PAIRWISE_BASED":
            nr = kw["neg_rate"]
            data = [rng.randint(400, size=B), rng.randint(6, size=B), rng.randint(400, size=B),
                    rng.randint(400, size=B * nr), rng.randint(6, size=B * nr), rng.randint(400, size=B * nr)]
        else:
            data = [rng.randint(400, size=B), rng.randint(6, size=B), rng.randint(400, size=B),
                    np.where(np.arange(B) % 2 == 0, 1, -1)]
        la, lb = a.train_batch(data), b.train_batch(data)
        assert abs(la - lb) <= 1e-4 * max(abs(lb), 1e-6), (step, la, lb)
        for (ka, va), (kb, vb) in zip(a.model.state_dict().items(), b.model.state_dict().items()):
            diff = (va - vb).abs()
            if opt == "sgd" and model_name != "kg2e":
                assert float(diff.max()) <= atol, (ka, step, float(diff.max()))
            else:
                # Both modes sum the row gradients with unordered float atomics, so they agree to rounding only.
                # Adagrad and Adam divide by a gradient magnitude: an element whose contributions cancel to ~0 can
                # step by about +-lr in different directions in the two modes.  The hinge's gradient jumps at
                # v = 0: from the second step on, a pair within rounding of the margin can be active in one mode
                # only (seen with KG2E at the third step, 5e-4 apart).  All but a handful of elements must agree
                # within atol, and none may be further apart than 2 lr per step taken.
                assert float((diff > atol).float().mean()) <= 1e-3, (ka, step, float((diff > atol).float().mean()))
                assert float(diff.max()) <= 2 * kw["learning_rate"] * (step + 1), (ka, step, float(diff.max()))


def test_evaluator_matches_oracle_and_reference_metrics():
    """Evaluator.test (batched rank kernel) == oracle rank counts; settle() metrics follow."""
    import oracle
    from oracle import ref_port
    from pykg2vec_b200.synthetic import SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(600, 5, 3000, 40, 30, seed=5)
    tr = _trainer_for("complex", kg, hidden_size=32, lmbda=0.1)
    ev = tr.evaluator
    res = ev.full_test(epoch=0)
    tabs = [w.detach().cpu().numpy() for w in tr.model.kge_tables()]
    om = oracle.Model("complex", tabs, 32)
    test = kg.arrays["test"]
    from pykg2vec_b200.evaluator import build_filter_csr
    hr_t, tr_h = kg.read_cache_data("hr_t"), kg.read_cache_data("tr_h")
    ft = build_filter_csr([(int(h), int(r)) for h, r, t in test], hr_t)
    fh = build_filter_csr([(int(t), int(r)) for h, r, t in test], tr_h)
    want = oracle.rank_1vsall(om, test[:, 0], test[:, 1], test[:, 2], ft, fh)
    mc = ev.metric_calculator
    got = np.stack([mc.rank_tail, mc.f_rank_tail, mc.rank_head, mc.f_rank_head], axis=1)
    np.testing.assert_array_equal(got, want)
    ref = ref_port.settle(want)
    assert res["mr"] == pytest.approx(ref["mr"]) and res["fmrr"] == pytest.approx(ref["fmrr"])
    # infer-style single query API: descending score order, length topk (evaluator.py:249-260)
    top = ev.test_tail_rank(int(test[0, 0]), int(test[0, 1]), topk=5)
    assert top.shape == (5,)
    full = oracle.sweep_scores(om, oracle.GROUP_TAIL, int(test[0, 0]), int(test[0, 1]), 0)
    assert set(top.cpu().tolist()) == set(np.argsort(-full, kind="stable")[:5].tolist())


def test_rescal_model_normalises_in_place_like_reference():
    """Rescal.forward mutates its tables (pairwise.py:843-844): rows become unit-norm, then scores
    match the oracle on the normalised tables; backward reaches both tables."""
    import oracle
    import pykg2vec_b200
    torch.manual_seed(3)
    m = pykg2vec_b200.import_model("rescal")(tot_entity=90, tot_relation=4, hidden_size=20, margin=1.0).cuda()
    before = [w.detach().cpu().numpy().copy() for w in m.kge_tables()]
    rng = np.random.RandomState(0)
    h, r, t = rng.randint(90, size=40), rng.randint(4, size=40), rng.randint(90, size=40)
    s = m(_cuda(h), _cuda(r), _cuda(t))
    want_tabs = [oracle.normalize_rows(b.copy()) for b in before]
    for w, wt in zip(m.kge_tables(), want_tabs):
        np.testing.assert_array_equal(w.detach().cpu().numpy(), wt)
    om = oracle.Model("rescal", want_tabs, 20)
    np.testing.assert_array_equal(gpu.bits(s.detach().cpu().numpy()), gpu.bits(oracle.score_fwd(om, h, r, t)))
    s.sum().backward()
    assert all(w.grad is not None and float(w.grad.abs().sum()) > 0 for w in m.kge_tables())


def test_device_sampler_matches_oracle_and_rules():
    """kge_sample_negatives == oracle bit-for-bit; negatives never hit a positive; layout and
    labels follow generator.py:42-158; Bernoulli probabilities steer the corrupted side."""
    import oracle
    L = _L()
    rng = np.random.RandomState(0)
    N, R, n_train = 60, 4, 2500  # dense graph: rejections do happen
    train = np.unique(np.stack([rng.randint(N, size=n_train), rng.randint(R, size=n_train),
                                rng.randint(N, size=n_train)], 1), axis=0)
    slots = L.tripleset_build(_cuda(train[:, 0].copy()), _cuda(train[:, 1].copy()), _cuda(train[:, 2].copy()), N, R)
    B = 300
    sel = rng.randint(len(train), size=B)
    ph, pr, pt = train[sel, 0].copy(), train[sel, 1].copy(), train[sel, 2].copy()
    positives = set(map(tuple, train.tolist()))
    for neg_rate, probs in ((1, None), (4, np.array([0.05, 0.5, 0.95, 0.3], dtype=np.float32))):
        hp = _cuda(probs) if probs is not None else None
        nh, nr, nt = L.sample_negatives(slots, _cuda(ph), _cuda(pr), _cuda(pt), neg_rate, hp, N, seed=7, step=3)
        want = oracle.sample_negatives(train, ph, pr, pt, neg_rate, probs, N, 7, 3)
        for a, b in zip((nh, nr, nt), want):
            np.testing.assert_array_equal(a.cpu().numpy(), b)
        nh, nr, nt = nh.cpu().numpy(), nr.cpu().numpy(), nt.cpu().numpy()
        rep_h, rep_t = np.repeat(ph, neg_rate), np.repeat(pt, neg_rate)
        assert np.array_equal(nr, np.repeat(pr, neg_rate))
        assert all((nh[i] == rep_h[i]) or (nt[i] == rep_t[i]) for i in range(len(nh)))  # one side kept
        assert not any((int(a), int(b), int(c)) in positives for a, b, c in zip(nh, nr, nt))
        if probs is not None:
            head_corrupted = nt == rep_t
            r_rep = np.repeat(pr, neg_rate)
            assert head_corrupted[r_rep == 2].mean() > 0.8 and head_corrupted[r_rep == 0].mean() < 0.2
        # pointwise layout: each positive followed by its negatives, labels +1/-1
        h4, r4, t4, y4 = L.sample_negatives(slots, _cuda(ph), _cuda(pr), _cuda(pt), neg_rate, hp, N, seed=7, step=3, layout=1)
        w4 = oracle.sample_negatives(train, ph, pr, pt, neg_rate, probs, N, 7, 3, layout=1)
        for a, b in zip((h4, r4, t4, y4), w4):
            np.testing.assert_array_equal(a.cpu().numpy(), b)
        y = y4.cpu().numpy().reshape(B, 1 + neg_rate)
        assert (y[:, 0] == 1).all() and (y[:, 1:] == -1).all()
        assert np.array_equal(h4.cpu().numpy().reshape(B, -1)[:, 0], ph)
    # a different step gives a different draw
    a = L.sample_negatives(slots, _cuda(ph), _cuda(pr), _cuda(pt), 1, None, N, seed=7, step=4)
    b = L.sample_negatives(slots, _cuda(ph), _cuda(pr), _cuda(pt), 1, None, N, seed=7, step=3)
    assert not (torch.equal(a[0], b[0]) and torch.equal(a[2], b[2]))


def test_generator_feeds_trainer_epoch():
    from pykg2vec_b200.generator import Generator, relation_property
    from pykg2vec_b200.synthetic import SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(300, 5, 4000, 50, 50, seed=3)
    for model_name, opt in (("transe", "sgd"), ("distmult", "adagrad")):
        tr = _trainer_for(model_name, kg, optimizer=opt, learning_rate=0.05, hidden_size=32, margin=1.0,
                          l1_flag=False, lmbda=0.01, batch_size=256, neg_rate=2 if model_name == "distmult" else 1,
                          sampling="bern")
        gen = Generator(tr.model, tr.config, seed=1)
        assert gen.head_prob is not None and gen.head_prob.shape[0] == 5
        before = [w.detach().clone() for w in tr.model.kge_tables()]
        loss = tr.train_model_epoch(gen, num_batch=5)
        assert np.isfinite(loss) and loss > 0
        assert any(not torch.equal(a, b.detach()) for a, b in zip(before, tr.model.kge_tables()))
        gen.start_one_epoch(1)
        batch = next(gen)
        assert len(batch) == (6 if model_name == "transe" else 4) and all(x.is_cuda for x in batch)
        with pytest.raises(StopIteration):
            next(gen)
    p = relation_property(kg.arrays["train"], 5)
    assert p.shape == (5,) and ((p > 0) & (p < 1)).all()


def test_convkb_trains_like_the_written_chain():
    """ConvKB (kernel on the collapsed affine form) follows the as-written conv -> concat -> Linear
    chain through whole optimizer steps: same loss and same updated parameters as torch autograd
    on oracle.ref_port's restatement, with the convolution filters left untouched (they are not
    registered parameters in the reference either, pointwise.py:280)."""
    import pykg2vec_b200
    from oracle import ref_port
    from pykg2vec_b200.criterion import Criterion
    g = gu.load("convkb_d24")
    m = _make_model(g)
    raw = [torch.from_numpy(x.astype(np.float64)) for x in gu.raw_tables_of(g)]
    train_idx = [0, 1, len(raw) - 2, len(raw) - 1]          # ent, rel, fc1.weight, fc1.bias
    params = [raw[i].clone().requires_grad_() for i in train_idx]
    opt_ref = torch.optim.SGD(params, lr=0.05)
    opt = torch.optim.SGD(m.parameters(), lr=0.05)
    assert len(list(m.parameters())) == 4
    conv_before = [c.weight.detach().clone() for c in m.conv_list]
    h, r, t = g["h"], g["r"], g["t"]
    y = np.where(np.arange(len(h)) % 2 == 0, 1.0, -1.0).astype(np.float32)
    for step in range(3):
        tabs = list(raw)
        for i, p in zip(train_idx, params):
            tabs[i] = p
        s_ref = ref_port.score("convkb_raw", tabs, torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t))
        loss_ref = ref_port.pointwise_logistic(s_ref, torch.from_numpy(y).double())
        opt_ref.zero_grad(); loss_ref.backward(); opt_ref.step()
        loss = Criterion.pointwise_logistic(m(_cuda(h), _cuda(r), _cuda(t)), _cuda(y)) + m.get_reg(None, None, None)
        opt.zero_grad(); loss.backward(); opt.step()
        assert abs(loss.item() - loss_ref.item()) <= 2e-5 * abs(loss_ref.item())
    got = [m.ent_embeddings.weight, m.rel_embeddings.weight, m.fc1.weight, m.fc1.bias]
    for a, b in zip(got, params):
        np.testing.assert_allclose(a.detach().cpu().numpy(), b.detach().numpy(), rtol=2e-4, atol=2e-6)
    for c, w0 in zip(m.conv_list, conv_before):
        assert torch.equal(c.weight.detach(), w0)


def test_train_batch_async_handle_equals_sync():
    """train_batch(sync=False) enqueues the same graph-staged step and hands back the loss lazily:
    identical losses and weights to the synchronous calls."""
    from pykg2vec_b200.synthetic import SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(400, 6, 2000, 50, 50, seed=1)
    kw = dict(optimizer="sgd", learning_rate=0.05, hidden_size=64, margin=1.0, l1_flag=False, neg_rate=1)
    a = _trainer_for("transe", kg, fused_step=True, **kw)
    b = _trainer_for("transe", kg, fused_step=True, **kw)
    b.model.load_state_dict(a.model.state_dict())
    rng = np.random.RandomState(4)
    B = 128
    batches = [[rng.randint(400, size=B), rng.randint(6, size=B), rng.randint(400, size=B),
                rng.randint(400, size=B), rng.randint(6, size=B), rng.randint(400, size=B)] for _ in range(4)]
    want = [a.train_batch(d) for d in batches]
    got = []
    for d in batches:
        h = b.train_batch(d, sync=False)      # enqueued only
        _ = sum(int(x.sum()) for x in d)      # host work overlapping the step
        got.append(float(h))                  # waits for this step's D2H (the handle is valid until the next call)
    # (the loss and the row gradients are accumulated with float atomics: equal up to summation order)
    np.testing.assert_allclose(got, want, rtol=1e-5)
    for (ka, va), (kb, vb) in zip(a.model.state_dict().items(), b.model.state_dict().items()):
        np.testing.assert_allclose(va.cpu().numpy(), vb.cpu().numpy(), rtol=0, atol=2e-6, err_msg=ka)
