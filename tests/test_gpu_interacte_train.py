"""InteractE's training-mode trunk on the device (kge_interacte_train_* of include/kge_b200.h) and every layer above
it: the forward's fixed-order statistics (bit-equal to the CPU oracle on the goldens and at the FB15k-237 shape of all
three yaml geometries, each group independent of the others, two groups in one call = two sequential calls), the
forward and backward against an fp64 autograd restatement of the formulas, the autograd Function against the
reference's torch layers fed the same noise, the Trainer's fused step against loss.backward() + torch.optim on the
torch layers, dropout runs that learn and repeat under a seed, the Evaluator after fused training, the step's peak
memory, and no cuDNN convolution in a training step.  The reference's own training-step numbers are checked by
tests/test_gpu_interacte.py, which now runs through these kernels."""
import types

import numpy as np
import pytest
import torch

import interacte_train_util as itu

pytestmark = pytest.mark.gpu

YAML = [(1, 96, 9, 20, 10), (2, 96, 11, 20, 10), (4, 64, 7, 20, 10)]   # (P, F, ks, rh, rw) of InteractE.yaml
# (N, R, geometry, B): the default yaml geometry at a modest N, and a small odd geometry with P = 3
SHAPES = [(300, 11, YAML[0], 32), (60, 5, (3, 5, 7, 6, 4), 7)]
FB237 = dict(N=14541, R=237)


def _model(N, R, geom, drops=(0.0, 0.0, 0.0), kge_trunk=True, seed=0):
    from pykg2vec_b200 import import_model
    P, F, ks, rh, rw = geom
    torch.manual_seed(seed)
    np.random.seed(seed)
    m = import_model("interacte")(tot_entity=N, tot_relation=R, hidden_size=rh * rw, input_dropout=drops[0],
                                  feature_map_dropout=drops[1], hidden_dropout=drops[2], feature_permutation=P,
                                  num_filters=F, kernel_size=ks, reshape_height=rh, reshape_width=rw, device="cuda",
                                  kge_trunk=kge_trunk)
    with torch.no_grad():   # BatchNorms away from their identity initialisation
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
    return m.cuda().train()


def _load(sd, N, R, drops=(0.0, 0.0, 0.0)):
    """the package's InteractE holding a numpy state (with "_geometry" and "_perm")"""
    m = _model(N, R, tuple(int(v) for v in sd["_geometry"]), drops)
    m.load_state_dict({key: torch.from_numpy(np.asarray(v)) for key, v in sd.items() if not key.startswith("_")},
                      strict=True)
    m.chequer_perm = torch.from_numpy(np.asarray(sd["_perm"], np.int64)).cuda()
    return m.cuda().train()


def _ids(N, R, B, seed):
    g = torch.Generator().manual_seed(seed)
    e, r = torch.randint(0, N, (B,), generator=g), torch.randint(0, R, (B,), generator=g)
    e[1], r[2] = e[0], r[0]   # ids repeat within the batch: the scatter into the tables must accumulate
    return e.cuda(), r.cuda()


def _widths(geom):
    P, F, ks, rh, rw = geom
    return P * 2 * rh * rw, P * F, rh * rw


def _noise(B, geom, p=(0.2, 0.5, 0.3), seed=5):
    g = torch.Generator("cuda").manual_seed(seed)
    return [(torch.rand(B, w, device="cuda", generator=g) >= q).float() / (1 - q)
            for w, q in zip(_widths(geom), p)]


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _running(m):
    return [t.clone() for bn in (m.bn0, m.bn1, m.bn2) for t in (bn.running_mean, bn.running_var)]


@pytest.mark.parametrize("name", itu.CASES)
def test_forward_kernels_equal_oracle_bitwise_on_goldens(name):
    """the tail and head forwards of a golden case as one call of two groups, with the reference's noise: x and the
    running statistics equal the CPU oracle (tests/oracle_interacte_train) bit for bit"""
    from pykg2vec_b200 import _lib
    g = itu.load(name)
    sd = itu.state(g)
    m = _load(sd, int(g["N"]), int(g["R"]))
    B = len(g["h"])
    e, r = np.concatenate([g["h"], g["t"]]), np.concatenate([g["r"], g["r"]])
    nz = [None if a is None else np.concatenate([a, b]) for a, b in zip(itu.noises(g, "tail"), itu.noises(g, "head"))]
    run = {}
    want = itu.oracle_fwd(sd, e, r, B, *nz, running=run)
    x, _ = _lib.interacte_train_fwd(m, torch.from_numpy(e).cuda(), torch.from_numpy(r).cuda(), B,
                                    *[None if a is None else torch.from_numpy(a).cuda() for a in nz])
    assert _bits_equal(x.cpu(), torch.from_numpy(want))
    sd_after = m.state_dict()
    for key in itu.RUNNING:
        assert _bits_equal(sd_after[key].cpu(), torch.from_numpy(run[key])), key


@pytest.mark.parametrize("geom", YAML, ids=lambda g: "P%d_F%d_ks%d" % g[:3])
def test_forward_kernels_equal_oracle_bitwise_at_fb15k237_shape(geom):
    """N = 14,541, R = 237, the two directions of B = 128 in one call, with dropout noise, at each yaml geometry"""
    from pykg2vec_b200 import _lib
    st = itu.random_state(FB237["N"], FB237["R"], geom, seed=11)
    m = _load(st, **FB237)
    B = 128
    e, r = _ids(FB237["N"], FB237["R"], 2 * B, 6)
    nz = _noise(2 * B, geom)
    run = {}
    want = itu.oracle_fwd(st, e.cpu().numpy(), r.cpu().numpy(), B, *[n.cpu().numpy() for n in nz], running=run)
    x, _ = _lib.interacte_train_fwd(m, e, r, B, *nz)
    assert _bits_equal(x.cpu(), torch.from_numpy(want)) and (x > 0).any()
    sd_after = m.state_dict()
    for key in itu.RUNNING:
        assert _bits_equal(sd_after[key].cpu(), torch.from_numpy(run[key])), key


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "P%d_ks%d_B%d" % (s[2][0], s[2][2], s[3]))
def test_forward_is_reproducible_and_per_group(shape):
    """x of the tail and head rows in ONE call equals two separate calls bit for bit, repeats bit for bit, and the
    running statistics after the one call equal those after the two calls in order"""
    from pykg2vec_b200 import _lib
    N, R, geom, B = shape
    e, r = _ids(N, R, 2 * B, 1)
    nz = _noise(2 * B, geom)
    one, two = _model(N, R, geom), _model(N, R, geom)
    assert torch.equal(one.chequer_perm, two.chequer_perm)
    x, _ = _lib.interacte_train_fwd(one, e, r, B, *nz)
    xa, _ = _lib.interacte_train_fwd(two, e[:B].contiguous(), r[:B].contiguous(), B, *[n[:B].contiguous() for n in nz])
    xb, _ = _lib.interacte_train_fwd(two, e[B:].contiguous(), r[B:].contiguous(), B, *[n[B:].contiguous() for n in nz])
    assert _bits_equal(x, torch.cat([xa, xb]))
    for a, b in zip(_running(one), _running(two)):
        assert _bits_equal(a, b)
    again, _ = _lib.interacte_train_fwd(one, e, r, B, *nz, running=False)
    assert _bits_equal(x, again)


def _trunk64(m, P64, e, r, n0, n1, n2):
    """the training-mode trunk (projection.py:427-442) in float64 torch ops: x, and the six batch statistics"""
    P, F, ks, H, W = m.feature_permutation, m.num_filters, m.kernel_size, 2 * m.reshape_width, m.reshape_height
    pad, B = ks // 2, e.numel()
    ent, rel, w0, b0, filt, w1, b1, fw, fb, w2, b2 = P64

    def bn(v, dims, w, b, eps=1e-5):
        mean = v.mean(dims, keepdim=True)
        var = v.var(dims, unbiased=False, keepdim=True)
        return (v - mean) / torch.sqrt(var + eps) * w + b, mean.flatten(), var.flatten()

    comb = torch.cat([ent[e], rel[r]], dim=1)
    x = comb[:, m.chequer_perm].reshape(B, P, H, W)
    x, m0, v0 = bn(x, (0, 2, 3), w0.view(1, -1, 1, 1), b0.view(1, -1, 1, 1))
    x = x * n0.double().view(B, P, H, W)
    x = torch.cat([x[..., H - pad:, :], x, x[..., :pad, :]], dim=2)
    x = torch.cat([x[..., W - pad:], x, x[..., :pad]], dim=3)
    x = torch.nn.functional.conv2d(x, filt.repeat(P, 1, 1, 1), groups=P)
    x, m1, v1 = bn(x, (0, 2, 3), w1.view(1, -1, 1, 1), b1.view(1, -1, 1, 1))
    x = torch.relu(x) * n1.double().view(B, P * F, 1, 1)
    x = (x.reshape(B, -1) @ fw.t() + fb) * n2.double()
    x, m2, v2 = bn(x, (0,), w2, b2)
    return torch.relu(x), (m0, v0, m1, v1, m2, v2)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "P%d_ks%d_B%d" % (s[2][0], s[2][2], s[3]))
def test_forward_and_backward_match_fp64_autograd(shape):
    from pykg2vec_b200 import _lib
    N, R, geom, B = shape
    m = _model(N, R, geom)
    e, r = _ids(N, R, B, 2)
    nz = _noise(B, geom)
    params = m.kge_interacte_params()
    P64 = [p.detach().double().requires_grad_() for p in params]
    run0 = _running(m)
    x, ws = _lib.interacte_train_fwd(m, e, r, B, *nz)
    with torch.backends.cudnn.flags(enabled=False):
        want, stats = _trunk64(m, P64, e, r, *nz)
    assert (x.double() - want).abs().max().item() <= 2e-5 * want.abs().max().item()
    HW = 2 * geom[3] * geom[4]
    counts = (B * HW, B * HW, B)   # running statistics: (1 - 0.1) * old + 0.1 * batch, unbiased variance
    for i, (got, old) in enumerate(zip(_running(m), run0)):
        n = counts[i // 2]
        ref = 0.9 * old.double() + 0.1 * stats[i] * (n / (n - 1) if i % 2 else 1.0)
        assert (got.double() - ref).abs().max().item() <= 1e-5 * (1 + ref.abs().max().item()), i
    up = torch.randn(B, x.shape[1], device="cuda", generator=torch.Generator("cuda").manual_seed(7))
    (want * up.double()).sum().backward()
    grads = [torch.zeros_like(p) for p in params]
    _lib.interacte_train_bwd(m, e, r, B, up, x, grads, ws, *nz)
    scale = max(p.grad.abs().max().item() for p in P64)
    for name, got, p in zip(_lib.INTERACTE_TRAIN_PARAMS, grads, P64):
        # bn0 and fc.bias sit in front of a training-mode BatchNorm: their true gradient is ~0 and both sides hold
        # rounding noise, bounded relative to the largest gradient of the step
        assert (got.double() - p.grad).abs().max().item() <= 5e-4 * p.grad.abs().max().item() + 1e-5 * scale, name


class _Mul(torch.nn.Module):
    """a dropout module replaced by a fixed noise tensor"""

    def __init__(self, noise):
        super().__init__()
        self.noise = noise

    def forward(self, x):
        return x * self.noise


def test_function_matches_torch_layers_with_the_same_noise():
    """InteracteTrunkFunction against _trunk_layers whose three dropout modules multiply by the same noise: x, every
    gradient, the running statistics and num_batches_tracked"""
    from pykg2vec_b200.projection import InteracteTrunkFunction
    N, R, geom, B = SHAPES[0]
    P, F, ks, rh, rw = geom
    e, r = _ids(N, R, B, 3)
    nz = _noise(B, geom)
    up = torch.randn(B, rh * rw, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
    out = []
    for kernel in (True, False):
        m = _model(N, R, geom, drops=(0.2, 0.5, 0.3), kge_trunk=kernel)
        if kernel:
            x = InteracteTrunkFunction.apply(m, e, r, B, *nz, *m.kge_interacte_params())
            m.note_batch_stats()
        else:
            m.inp_drop = _Mul(nz[0].view(B, P, 2 * rw, rh))
            m.feature_map_drop = _Mul(nz[1].view(B, P * F, 1, 1))
            m.hidden_drop = _Mul(nz[2])
            x = m._trunk_layers(e, r)
        (x * up).sum().backward()
        out.append((x.detach(), [p.grad for p in m.kge_interacte_params()], m.state_dict()))
    (xa, ga, sa), (xb, gb, sb) = out
    assert (xa - xb).abs().max().item() <= 2e-5 * xb.abs().max().item()
    scale = max(g.abs().max().item() for g in gb)
    for a, b in zip(ga, gb):
        assert (a - b).abs().max().item() <= 5e-4 * b.abs().max().item() + 1e-5 * scale
    for key in sa:
        if "running" in key or "num_batches" in key:
            assert (sa[key].double() - sb[key].double()).abs().max().item() <= 1e-5, key


def _trainer(N, R, geom, opt, fused, drops=(0.0, 0.0, 0.0), lr=0.01):
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    m = _model(N, R, geom, drops=drops, kge_trunk=fused)
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
    h[1], r[3] = h[0], r[0]   # repeated ids
    hr_t, tr_h = np.zeros((B, N), np.float32), np.zeros((B, N), np.float32)
    hr_t[np.arange(B), t] = 1.0
    tr_h[np.arange(B), h] = 1.0
    hr_t[:, :3] = 1.0
    return [h, r, t, torch.from_numpy(hr_t), torch.from_numpy(tr_h)]


# in front of a training-mode BatchNorm with dropouts 0 their true gradient is ~0: bn0's affine parameters (the circular
# conv of a per-image constant is a per-channel constant, which bn1 removes; bn0's scale is normalised away likewise)
# and fc.bias (no ReLU between fc and bn2)
INVISIBLE = ("bn0.weight", "bn0.bias", "fc.bias")


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "P%d_ks%d_B%d" % (s[2][0], s[2][2], s[3]))
def test_fused_steps_match_autograd_on_torch_layers(opt, shape):
    """_fused_interacte against train_step_projection + loss.backward() + torch.optim on _trunk_layers, dropouts 0,
    three steps.  Adagrad and Adam divide each element's step by its own gradient magnitude, so rounding noise in a
    near-zero gradient moves the element by up to lr: the bounds are those of the ConvE and HypER training tests (SGD
    carries the comparison; under Adagrad / Adam at most 1% of the elements may differ by more than 1% of lr, and the
    INVISIBLE parameters, whose true gradient is 0 with dropouts 0, are held to 6 lr)."""
    N, R, geom, B = shape
    lr = 0.01
    a, b = _trainer(N, R, geom, opt, True, lr=lr), _trainer(N, R, geom, opt, False, lr=lr)
    assert a._interacte and not b._interacte and not b.model.kge_trunk
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
            assert diff.max().item() <= 6 * lr, key
            if key not in INVISIBLE:
                assert (diff > 5 * tol).float().mean().item() <= 1e-2, key
    sa, sb = a.model.state_dict(), b.model.state_dict()
    for key in sa:
        if "running" in key or "num_batches" in key:
            tol = 1e-4 if (opt == "sgd" or key.startswith("bn0")) else 6 * lr
            assert (sa[key].double() - sb[key].double()).abs().max().item() <= tol, key


def test_one_row_batch_raises_before_any_launch():
    from pykg2vec_b200 import _lib
    N, R, geom, _ = SHAPES[1]
    m = _model(N, R, geom)
    e, r = torch.tensor([5], device="cuda"), torch.tensor([1], device="cuda")
    before = (_lib.launch_count(), _running(m))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m(e, r)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        _trainer(N, R, geom, "adam", True).train_batch_device([e, r, e, torch.zeros(1, N, device="cuda"),
                                                               torch.zeros(1, N, device="cuda")])
    assert _lib.launch_count() == before[0]
    assert all(torch.equal(a, b) for a, b in zip(before[1], _running(m)))


def test_fused_steps_with_dropout_learn_and_repeat():
    N, R, geom, B = SHAPES[1]
    batch = _batch(N, R, 32, 9)
    runs = []
    for rep in range(2):
        tr = _trainer(N, R, geom, "adam", True, drops=(0.2, 0.5, 0.3), lr=0.01)
        torch.manual_seed(42)
        runs.append([tr.train_batch(batch) for _ in range(30)])
    assert np.isfinite(runs[0]).all() and np.mean(runs[0][-5:]) < np.mean(runs[0][:5])
    # the three dropouts follow torch.manual_seed: a reseeded run repeats up to the order of the float atomics
    assert np.allclose(runs[0][:3], runs[1][:3], rtol=1e-5, atol=0)
    tr = _trainer(N, R, geom, "adam", True, drops=(0.2, 0.5, 0.3), lr=0.01)
    torch.manual_seed(43)
    assert abs(tr.train_batch(batch) - runs[0][0]) > 1e-6 * runs[0][0]


def test_evaluator_after_fused_training_matches_the_torch_path():
    """after fused adam steps, the Evaluator's raw ranks (kge_interacte_trunk_fwd + kge_proj_rank) against ranks
    counted from the torch layers' predictions (eval mode) on the same weights"""
    from pykg2vec_b200.evaluator import Evaluator
    N, R, geom, B = SHAPES[0]
    tr = _trainer(N, R, geom, "adam", True, lr=0.003)
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


def _fb237_trainer(fused):
    return _trainer(FB237["N"], FB237["R"], YAML[0], "adam", fused, drops=(0.2, 0.5, 0.3), lr=0.0001)


def _fb237_batch(tr, B=128):
    batch = _batch(FB237["N"], FB237["R"], B, 3)
    return tr._projection_batch(batch)[0]


def test_fused_step_peak_memory_at_the_bench_shape():
    """one fused step at the FB15k-237 shape (B = 128, Adam, the default yaml geometry) allocates at most the trunk's
    workspace for 2B rows + 32 MB above the standing tensors: the [2B, N] predictions and one [B, N] gradient (22 MB),
    the noise and x / gx"""
    from pykg2vec_b200 import _lib
    tr = _fb237_trainer(True)
    ids = _fb237_batch(tr)
    tr.train_batch_device(ids)   # warm-up: the optimizer state and scratch exist from build_model on
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    tr.train_batch_device(ids)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ws = _lib.interacte_train_workspace_bytes(tr.model, 256, 128)
    assert 0 < ws and peak <= ws + (32 << 20), (peak, ws)


def test_training_steps_run_no_cudnn_convolution():
    """InteractE(...).train() with CUDA tables: neither the fused step nor loss.backward() through
    InteracteTrunkFunction launches a cuDNN / convolution kernel"""
    from torch.profiler import ProfilerActivity, profile
    for fused in (True, False):
        tr = _fb237_trainer(True)
        if not fused:
            tr._interacte = False   # the autograd path on the kernels: train_step_projection + loss.backward()
        ids = _fb237_batch(tr)
        tr.train_batch_device(ids)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.train_batch_device(ids)
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
        assert any("interacte_tr_" in n for n in names), names[:20]
        cudnn = ("cudnn", "xmma", "implicit_gemm", "conv2d", "convolution", "depthwise", "winograd", "fprop", "dgrad",
                 "wgrad")
        bad = [n for n in names if any(w in n.lower() for w in cudnn)]
        assert not bad, (fused, bad[:10])
