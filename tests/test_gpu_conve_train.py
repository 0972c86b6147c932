"""ConvE's training-mode trunk on the device (kge_conve_train_* of include/kge_b200.h) and every layer above it: the
forward's fixed-order statistics (bit-reproducible, each group independent of the others, two groups in one call =
two sequential calls), the forward and backward against an fp64 autograd restatement of the formulas, the autograd
Function against the reference's torch layers fed the same noise, the Trainer's fused step against loss.backward() +
torch.optim on the torch layers, dropout runs that learn and repeat under a seed, B = 1, the Evaluator after fused
training, and the unmodified reference Trainer driving the class.  The reference's own numbers (golden vectors) are
checked by tests/test_gpu_proj.py::test_conve_*, which now run through these kernels."""
import types

import numpy as np
import pytest
import torch

import dropin_util as du

pytestmark = pytest.mark.gpu

# (N, R, k, h1, B): the reference's 20 x 20 image at a modest N, and a 12 x 6 image (widths not multiples of 4)
SHAPES = [(300, 11, 200, 20, 64), (60, 5, 36, 6, 7)]


def _model(N, R, k, h1, drops=(0.0, 0.0, 0.0), kge_trunk=True, seed=0):
    from pykg2vec_b200 import import_model
    torch.manual_seed(seed)
    m = import_model("conve")(tot_entity=N, tot_relation=R, hidden_size=k, hidden_size_1=h1, lmbda=0.1,
                              input_dropout=drops[0], feature_map_dropout=drops[1], hidden_dropout=drops[2],
                              kge_trunk=kge_trunk)
    with torch.no_grad():   # BatchNorms away from their identity initialisation
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
    return m.cuda().train()


def _ids(N, R, B, seed, repeat=True):
    g = torch.Generator().manual_seed(seed)
    e, r = torch.randint(N, (B,), generator=g), torch.randint(2 * R, (B,), generator=g)
    if repeat:   # ids repeat within the batch: the scatter into the tables must accumulate
        e[1], r[2] = e[0], r[0]
    return e.cuda(), r.cuda()


def _noise(B, k, p=(0.2, 0.2, 0.3), seed=5):
    g = torch.Generator("cuda").manual_seed(seed)
    out = []
    for width, q in ((2 * k, p[0]), (32, p[1]), (k, p[2])):
        out.append((torch.rand(B, width, device="cuda", generator=g) >= q).float() / (1 - q))
    return out


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


@pytest.mark.parametrize("name", ["conve_train_k200_drop", "conve_train_12x6"])
def test_forward_kernels_equal_oracle_bitwise(name):
    """the tail and head forwards of a golden case as one call of two groups, with the reference's noise: x and the
    running statistics equal the CPU oracle (tests/oracle_conve_train) bit for bit"""
    import conve_train_util as cu
    from pykg2vec_b200 import _lib, import_model
    g = cu.load(name)
    sd, k, h1, R = cu.state(g), int(g["hidden_size"]), int(g["hidden_size_1"]), int(g["R"])
    m = import_model("conve")(tot_entity=int(g["N"]), tot_relation=R, hidden_size=k, hidden_size_1=h1, lmbda=0.1,
                              input_dropout=0.0, feature_map_dropout=0.0, hidden_dropout=0.0)
    m.load_state_dict({key: torch.from_numpy(np.asarray(v)) for key, v in sd.items()}, strict=True)
    m.cuda().train()
    B = len(g["h"])
    e, r = np.concatenate([g["h"], g["t"]]), np.concatenate([g["r"], g["r"] + R])
    nz = [None if a is None else np.concatenate([a, b]) for a, b in zip(cu.noises(g, "tail"), cu.noises(g, "head"))]
    run = {}
    want = cu.oracle_fwd(sd, k, h1, e, r, B, *nz, running=run)
    x, _ = _lib.conve_train_fwd(m, torch.from_numpy(e).cuda(), torch.from_numpy(r).cuda(), B,
                                *[None if a is None else torch.from_numpy(a).cuda() for a in nz])
    assert _bits_equal(x.cpu(), torch.from_numpy(want))
    sd_after = m.state_dict()
    for key in cu.RUNNING:
        assert _bits_equal(sd_after[key].cpu(), torch.from_numpy(run[key])), key


def _running(m):
    return [t.clone() for bn in (m.bn0, m.bn1, m.bn2) for t in (bn.running_mean, bn.running_var)]


class _Mul(torch.nn.Module):
    """a dropout module replaced by a fixed noise tensor"""

    def __init__(self, noise):
        super().__init__()
        self.noise = noise

    def forward(self, x):
        return x * self.noise


def _trunk64(m, e, r, n0, n1, n2):
    """the training-mode trunk (projection.py:86-99) in float64 torch ops: x, and the six batch statistics"""
    k, h1 = m.hidden_size, m.hidden_size_1
    h2, B = k // h1, e.numel()
    P = {n: p.double() for n, p in zip(("ent", "rel", "w0", "b0", "cw", "cb", "w1", "b1", "fw", "fb", "w2", "b2"),
                                       m._kge64)}

    def bn(v, dims, w, b, eps=1e-5):
        mean = v.mean(dims, keepdim=True)
        var = v.var(dims, unbiased=False, keepdim=True)
        return (v - mean) / torch.sqrt(var + eps) * w + b, mean.flatten(), var.flatten()

    x = torch.cat([P["ent"][e], P["rel"][r]], 1).view(B, 1, 2 * h2, h1)
    x, m0, v0 = bn(x, (0, 1, 2, 3), P["w0"].view(1, -1, 1, 1), P["b0"].view(1, -1, 1, 1))
    x = x * n0.double().view(B, 1, 2 * h2, h1)
    x = torch.nn.functional.conv2d(x, P["cw"], P["cb"])
    x, m1, v1 = bn(x, (0, 2, 3), P["w1"].view(1, -1, 1, 1), P["b1"].view(1, -1, 1, 1))
    x = torch.relu(x) * n1.double().view(B, 32, 1, 1)
    x = (x.reshape(B, -1) @ P["fw"].t() + P["fb"]) * n2.double()
    x, m2, v2 = bn(x, (0,), P["w2"], P["b2"])
    return torch.relu(x), (m0, v0, m1, v1, m2, v2)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "k%d_h1%d_B%d" % (s[2], s[3], s[4]))
def test_forward_is_reproducible_and_per_group(shape):
    """x of the tail and head rows in ONE call equals two separate calls bit for bit, repeats bit for bit, and the
    running statistics after the one call equal those after the two calls in order"""
    from pykg2vec_b200 import _lib
    N, R, k, h1, B = shape
    e, r = _ids(N, R, 2 * B, 1)
    nz = _noise(2 * B, k)
    one = _model(N, R, k, h1)
    two = _model(N, R, k, h1)
    x, _ = _lib.conve_train_fwd(one, e, r, B, *nz)
    xa, _ = _lib.conve_train_fwd(two, e[:B].contiguous(), r[:B].contiguous(), B, *[n[:B].contiguous() for n in nz])
    xb, _ = _lib.conve_train_fwd(two, e[B:].contiguous(), r[B:].contiguous(), B, *[n[B:].contiguous() for n in nz])
    assert _bits_equal(x, torch.cat([xa, xb]))
    for a, b in zip(_running(one), _running(two)):
        assert _bits_equal(a, b)
    again, _ = _lib.conve_train_fwd(one, e, r, B, *nz, running=False)
    assert _bits_equal(x, again)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "k%d_h1%d_B%d" % (s[2], s[3], s[4]))
def test_forward_and_backward_match_fp64_autograd(shape):
    from pykg2vec_b200 import _lib
    N, R, k, h1, B = shape
    m = _model(N, R, k, h1)
    e, r = _ids(N, R, B, 2)
    nz = _noise(B, k)
    params = m.kge_conve_params()
    m._kge64 = [p.detach().double().requires_grad_() for p in params]
    run0 = _running(m)
    x, ws = _lib.conve_train_fwd(m, e, r, B, *nz)
    want, stats = _trunk64(m, e, r, *nz)
    assert (x.double() - want).abs().max().item() <= 2e-5 * want.abs().max().item()
    # running statistics: (1 - 0.1) * old + 0.1 * batch, unbiased variance
    counts = (B * 2 * k, B * (2 * (k // h1) - 2) * (h1 - 2), B)
    for i, (got, old) in enumerate(zip(_running(m), run0)):
        n = counts[i // 2]
        batch = stats[i] * (n / (n - 1) if i % 2 else 1.0)
        ref = 0.9 * old.double() + 0.1 * batch
        assert (got.double() - ref).abs().max().item() <= 1e-5 * (1 + ref.abs().max().item()), i
    up = torch.randn(B, k, device="cuda", generator=torch.Generator("cuda").manual_seed(7))
    (want * up.double()).sum().backward()
    grads = [torch.zeros_like(p) for p in params]
    _lib.conve_train_bwd(m, e, r, B, up, x, grads, ws, *nz)
    scale = max(p.grad.abs().max().item() for p in m._kge64)
    for name, got, p in zip(_lib.CONVE_TRAIN_PARAMS, grads, m._kge64):
        ref = p.grad
        # conv bias and bn0 are invisible behind a training-mode BatchNorm: their true gradient is ~0 and both sides
        # hold rounding noise, bounded relative to the largest gradient of the step
        assert (got.double() - ref).abs().max().item() <= 5e-4 * ref.abs().max().item() + 1e-5 * scale, name


def test_function_matches_torch_layers_with_the_same_noise():
    """ConveTrunkFunction against _trunk_layers whose three dropout modules multiply by the same noise: x, every
    gradient, the running statistics and num_batches_tracked"""
    from pykg2vec_b200.projection import ConveTrunkFunction
    N, R, k, h1, B = SHAPES[0]
    e, r = _ids(N, R, B, 3)
    nz = _noise(B, k)
    up = torch.randn(B, k, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
    out = []
    for kernel in (True, False):
        m = _model(N, R, k, h1, drops=(0.2, 0.2, 0.3), kge_trunk=kernel)
        if kernel:
            x = ConveTrunkFunction.apply(m, e, r, B, *nz, *m.kge_conve_params())
            m.note_batch_stats()
        else:
            m.inp_drop = _Mul(nz[0].view(B, 1, 2 * (k // h1), h1))
            m.feat_drop = _Mul(nz[1].view(B, 32, 1, 1))
            m.hidden_drop = _Mul(nz[2])
            x = m._trunk_layers(e, r)
        (x * up).sum().backward()
        out.append((x.detach(), [p.grad for p in m.kge_conve_params()], m.state_dict()))
    (xa, ga, sa), (xb, gb, sb) = out
    assert (xa - xb).abs().max().item() <= 2e-5 * xb.abs().max().item()
    scale = max(g.abs().max().item() for g in gb)
    for a, b in zip(ga, gb):
        assert (a - b).abs().max().item() <= 5e-4 * b.abs().max().item() + 1e-5 * scale
    for key in sa:
        if "running" in key or "num_batches" in key:
            assert (sa[key].double() - sb[key].double()).abs().max().item() <= 1e-5, key


def test_one_row_batch_raises_before_any_launch():
    from pykg2vec_b200 import _lib
    m = _model(60, 5, 36, 6)
    e, r = _ids(60, 5, 1, 4, repeat=False)
    before = (_lib.launch_count(), _running(m))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m(e, r)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        _trainer(60, 5, 36, 6, "adam", True).train_batch_device([e, r, e, torch.zeros(1, 60, device="cuda"),
                                                                 torch.zeros(1, 60, device="cuda")])
    assert _lib.launch_count() == before[0]
    assert all(torch.equal(a, b) for a, b in zip(before[1], _running(m)))


def _trainer(N, R, k, h1, opt, fused, drops=(0.0, 0.0, 0.0), lr=0.01):
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    m = _model(N, R, k, h1, drops=drops, kge_trunk=fused)
    cfg = types.SimpleNamespace(device="cuda", optimizer=opt, learning_rate=lr, fused_step=fused, label_smoothing=0.1,
                                tot_entity=N, batch_size=16, knowledge_graph=None)
    tr = Trainer(m, cfg)
    ev, trmod.Evaluator = trmod.Evaluator, (lambda *a, **kw: None)   # no evaluation: no knowledge graph here
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev
    return tr


def _batch(N, R, B, seed):
    rng = np.random.RandomState(seed)
    h, r, t = rng.randint(N, size=B), rng.randint(R, size=B), rng.randint(N, size=B)
    h[1] = h[0]
    hr_t, tr_h = np.zeros((B, N), np.float32), np.zeros((B, N), np.float32)
    hr_t[np.arange(B), t] = 1.0
    tr_h[np.arange(B), h] = 1.0
    hr_t[:, :3] = 1.0
    return [h, r, t, torch.from_numpy(hr_t), torch.from_numpy(tr_h)]


# in front of a training-mode BatchNorm (bn1 / bn2) with dropouts 0: their true gradient is ~0
INVISIBLE = ("bn0.weight", "bn0.bias", "conv2d_1.bias", "fc.bias")


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "k%d_h1%d_B%d" % (s[2], s[3], s[4]))
def test_fused_steps_match_autograd_on_torch_layers(opt, shape):
    """_fused_conve against train_step_projection + loss.backward() + torch.optim on _trunk_layers, dropouts 0, three
    steps.  Adagrad and Adam divide each element's step by its own gradient magnitude, so rounding noise in a
    near-zero gradient moves the element by up to lr.  For bn0.*, conv2d_1.bias and fc.bias (true gradient 0 with
    dropouts 0) the bound of 2 lr per step is only a sanity check: two Adam runs cannot differ by more.  The SGD case
    and, under Adagrad / Adam, the rule that at most 1% of the other parameters' elements may differ by more than 1% of
    lr carry the comparison (Adagrad's first step is +-lr for ANY nonzero gradient: seen 7 of 4,400 relation
    elements)."""
    N, R, k, h1, B = shape
    lr = 0.01
    a, b = _trainer(N, R, k, h1, opt, True, lr=lr), _trainer(N, R, k, h1, opt, False, lr=lr)
    assert a._conve and not b._conve and not b.model.kge_trunk
    for step in range(3):
        batch = _batch(N, R, B, step)
        la, lb = a.train_batch(batch), b.train_batch(batch)
        assert abs(la - lb) <= 1e-4 * abs(lb)
    for (key, pa), pb in zip(a.model.named_parameters(), b.model.parameters()):
        diff, wb = (pa.detach() - pb.detach()).abs(), pb.detach()
        tol = 2e-3 * lr + 1e-5 * wb.abs().max().item()
        if opt == "sgd":
            assert diff.max().item() <= tol, key
        else:
            # an element whose gradient is near 0 steps by up to lr per step on either side's rounding (the backward's
            # float atomics run in no fixed order): bounded by 2 lr per step, and rare outside the invisible parameters
            assert diff.max().item() <= 6 * lr, key
            if key not in INVISIBLE:
                assert (diff > 5 * tol).float().mean().item() <= 1e-2, key
    # bn1's and bn2's running statistics see conv2d_1.bias, fc.bias and bn0's affine parameters directly: under
    # Adagrad / Adam they inherit those parameters' drift (momentum 0.1 of it per forward)
    sa, sb = a.model.state_dict(), b.model.state_dict()
    for key in sa:
        if "running" in key or "num_batches" in key:
            tol = 1e-4 if (opt == "sgd" or key.startswith("bn0")) else 6 * lr
            assert (sa[key].double() - sb[key].double()).abs().max().item() <= tol, key


def test_fused_steps_with_dropout_learn_and_repeat():
    N, R, k, h1, B = SHAPES[1]
    batch = _batch(N, R, 32, 9)
    runs = []
    for rep in range(2):
        tr = _trainer(N, R, k, h1, "adam", True, drops=(0.2, 0.2, 0.3), lr=0.01)
        torch.manual_seed(42)
        runs.append([tr.train_batch(batch) for _ in range(30)])
    assert np.isfinite(runs[0]).all() and np.mean(runs[0][-5:]) < np.mean(runs[0][:5])
    # the three dropouts follow torch.manual_seed: a reseeded run repeats up to the order of the float atomics
    assert np.allclose(runs[0][:3], runs[1][:3], rtol=1e-5, atol=0)
    tr = _trainer(N, R, k, h1, "adam", True, drops=(0.2, 0.2, 0.3), lr=0.01)
    torch.manual_seed(43)
    assert abs(tr.train_batch(batch) - runs[0][0]) > 1e-6 * runs[0][0]


def test_evaluator_after_fused_training_matches_the_torch_path():
    """after fused adam steps, the Evaluator's raw ranks (kge_conve_trunk_fwd + kge_proj_rank) against ranks counted
    from the torch layers' predictions (eval mode) on the same weights"""
    from pykg2vec_b200.evaluator import Evaluator
    N, R, k, h1, B = SHAPES[0]
    tr = _trainer(N, R, k, h1, "adam", True, lr=0.003)
    for step in range(5):
        tr.train_batch(_batch(N, R, B, 20 + step))
    m = tr.model.eval()
    ev = object.__new__(Evaluator)
    ev.model, ev.config = m, types.SimpleNamespace(device="cuda", tot_entity=N)
    ev._filter_cache, ev._workspace = {}, None
    rng = np.random.RandomState(2)
    h, r, t = rng.randint(N, size=100), rng.randint(R, size=100), rng.randint(N, size=100)
    with torch.no_grad():
        got = ev.rank_triples(h, r, t)
    hd, rd, td = (torch.from_numpy(a).cuda() for a in (h, r, t))
    with torch.enable_grad():
        pt = m(hd, rd, direction="tail").detach()   # grad-enabled eval forward: the torch layers
        ph = m(td, rd, direction="head").detach()
    ar = torch.arange(100, device="cuda")
    want_t = (pt > pt[ar, td][:, None]).sum(1).cpu().numpy()
    want_h = (ph > ph[ar, hd][:, None]).sum(1).cpu().numpy()
    assert np.mean(got[:, 0] == want_t) >= 0.97 and np.mean(got[:, 2] == want_h) >= 0.97
    assert np.abs(got[:, 0] - want_t).max() <= 2 and np.abs(got[:, 2] - want_h).max() <= 2


DROPIN_FLOW = r"""
import json, os, sys
import numpy as np
import torch
import dropin_util as du
B200Importer = du.b200_importer_class()
ds = du.write_dataset(os.path.abspath("data"))
argv = ["-mn", "conve", "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1", "-ds", "syn", "-dsp", ds,
        "-device", "cuda", "-k", "40", "-k2", "8", "-b", "32"]
tr = du.run_cli_flow(argv, B200Importer)
out = {"cls": type(tr.model).__module__ + "." + type(tr.model).__name__, "cuda": next(tr.model.parameters()).is_cuda,
       "kernels": bool(tr.model.kge_train_supported()),
       "tracked": int(tr.model.bn2.num_batches_tracked),
       "losses": [float(v) for _, v in tr.training_results],
       "mr_finite": all(bool(np.isfinite(v)) for v in tr.evaluator.metric_calculator.mr.values())}
print("RESULT " + json.dumps(out))
"""


@pytest.mark.skipif(not du.reference_available(), reason="oracle/_ref not installed (no reference checkout at build())")
def test_reference_trainer_drives_conve(tmp_path):
    """the unmodified reference CLI flow (Importer -> Trainer.build_model / train_model -> Evaluator) with this
    package's ConvE patched into Importer, -device cuda: loss.backward() and torch.optim train through the kernels"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", DROPIN_FLOW], cwd=str(tmp_path), env=env, capture_output=True,
                         text=True, timeout=300)
    lines = [ln for ln in res.stdout.splitlines() if ln.startswith("RESULT ")]
    assert res.returncode == 0 and lines, res.stderr[-4000:]
    out = json.loads(lines[-1][len("RESULT "):])
    assert out["cls"] == "pykg2vec_b200.projection.ConvE" and out["cuda"] and out["kernels"]
    assert out["tracked"] > 0 and len(out["losses"]) == 2 and np.isfinite(out["losses"]).all()
    assert out["mr_finite"]
