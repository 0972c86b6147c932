"""AcrE's training-mode trunk on the device (kge_acre_train_* of include/kge_b200.h) and every layer above it: the
forward's fixed-order statistics (bit-reproducible, each group independent of the others, two groups in one call = two
sequential calls), the forward and backward against an fp64 autograd restatement of the formulas for both ways
(with and without conv biases, atrous rates beyond the image), the autograd Function against the reference's torch
layers fed the same noise, the Trainer's fused step against loss.backward() + torch.optim on the torch layers, dropout
runs that learn and repeat under a seed, the Evaluator after fused training, the step's peak memory, and no cuDNN
convolution in a training step.  The reference's own training-step numbers are checked by tests/test_gpu_acre.py,
which now runs through these kernels."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import acre_train_util as atu
import acre_util as au

pytestmark = pytest.mark.gpu

# (N, R, way, C, atrous, acre_bias, B): the FB15k-237 configurations of acre_util at a modest N, and small ones with
# rates beyond the 20 x 20 image and no conv bias
SHAPES = [(300, 11, "serial", 32, (1, 2, 2), True, 32), (300, 11, "parallel", 9, (1, 2, 2), True, 32),
          (300, 11, "parallel", 32, (1, 3, 5), False, 16),
          (60, 5, "parallel", 5, (2, 11, 23), False, 7), (60, 5, "serial", 6, (1, 7, 21), False, 9)]
FB237 = dict(N=14541, R=237)


def _model(N, R, way, C, atrous, bias, drops=(0.0, 0.0, 0.0), kge_trunk=True, seed=0):
    from pykg2vec_b200 import import_model
    torch.manual_seed(seed)
    m = import_model("acre")(tot_entity=N, tot_relation=R, hidden_size=200, input_dropout=drops[0],
                             feature_map_dropout=drops[1], hidden_dropout=drops[2], in_channels=C, way=way,
                             first_atrous=atrous[0], second_atrous=atrous[1], third_atrous=atrous[2], acre_bias=bias,
                             kge_trunk=kge_trunk)
    with torch.no_grad():   # BatchNorms away from their identity initialisation
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
    return m.cuda().train()


def _shape_model(shape, **kw):
    N, R, way, C, atrous, bias, _ = shape
    return _model(N, R, way, C, atrous, bias, **kw)


def _ids(N, R, Q, seed):
    g = torch.Generator().manual_seed(seed)
    e, r = torch.randint(0, N, (Q,), generator=g), torch.randint(0, R, (Q,), generator=g)
    e[1], r[2] = e[0], r[0]   # ids repeat within the batch: the scatter into the tables must accumulate
    e[3] = e[4] = 7           # ... and one entity serves twice
    return e.cuda(), r.cuda()


def _noise(Q, C, p=(0.3, 0.2, 0.5), seed=5):
    g = torch.Generator("cuda").manual_seed(seed)
    return [(torch.rand(Q, w, device="cuda", generator=g) >= q).float() / (1 - q) for w, q in zip((400, C, 200), p)]


def _bits_equal(a, b):
    return torch.equal(a.view(torch.int32), b.view(torch.int32))


def _running(m):
    return [t.clone() for bn in (m.bn0, m.bn1, m.bn2) for t in (bn.running_mean, bn.running_var)]


# bn1 outputs within this fraction of their largest magnitude of 0 are "ambiguous": the fp32 forward may put one on
# the other side of the ReLU, which moves W_gate_e's / the convs' gradients by that element's whole share
AMBIGUOUS = 2e-6


def _relu_amb(z, g, flip):
    """ReLU of group g's bn1 output z, the mask of element flip = (group, flat index) toggled (None: the plain ReLU)"""
    if flip is None or flip[0] != g:
        return F.relu(z)
    mask = (z > 0).to(z.dtype)
    mask.view(-1)[flip[1]] = 1 - mask.view(-1)[flip[1]]
    return z * mask


def _trunk64(m, P, e, r, B, n0, n1, n2, running=None, flip=None, ambiguous=None):
    """fp64 restatement of the training-mode trunk (projection.py:706-734) over G groups of B rows with explicit noise;
    P: the kge_acre_params() tensors in fp64 (leaves).  running: six fp64 running-statistic tensors to update.  flip:
    (group, flat index) of one bn1 output whose ReLU mask is toggled; ambiguous: a list that gets bn1's ambiguous
    outputs as (group, flat index)."""
    names = [n for n in __import__("pykg2vec_b200")._lib.acre_train_present(m)]
    T = dict(zip(names, P))
    C = int(m.in_channels)
    rates = (m.first_atrous, m.second_atrous, m.third_atrous)
    xs = []
    for g in range(e.numel() // B):
        sl = slice(g * B, (g + 1) * B)
        img = torch.cat([T["ent"][e[sl]], T["rel"][r[sl]]], 1).view(-1, 1, 20, 20)
        rs = running or [None] * 6
        v = F.batch_norm(img, rs[0], rs[1], T["bn0_weight"], T["bn0_bias"], True, m.bn0.momentum, m.bn0.eps)
        if n0 is not None:
            v = v * n0[sl].double().view(-1, 1, 20, 20)

        def conv(l, x):
            return F.conv2d(x, T["conv%d_weight" % l], T.get("conv%d_bias" % l), 1, rates[l - 1], rates[l - 1])
        if m.way == "serial":
            y = conv(3, conv(2, conv(1, v))) + v
        else:
            gate = torch.cat([v.expand(-1, C, 20, 20).reshape(-1, C, 400)] +
                             [conv(l, v).reshape(-1, C, 400) for l in (1, 2, 3)], 2)
            y = F.linear(gate, T["W_gate_e_weight"], T["W_gate_e_bias"]).view(-1, C, 20, 20)
        z = F.batch_norm(y, rs[2], rs[3], T["bn1_weight"], T["bn1_bias"], True, m.bn1.momentum, m.bn1.eps)
        if ambiguous is not None:
            za = z.detach().abs().view(-1)
            ambiguous += [(g, int(i)) for i in torch.nonzero(za <= AMBIGUOUS * za.max()).view(-1)]
        f = _relu_amb(z, g, flip)
        if n1 is not None:
            f = f * n1[sl].double().view(-1, C, 1, 1)
        h = F.linear(f.reshape(f.shape[0], -1), T["fc_weight"], T["fc_bias"])
        if n2 is not None:
            h = h * n2[sl].double()
        xs.append(F.relu(F.batch_norm(h, rs[4], rs[5], T["bn2_weight"], T["bn2_bias"], True, m.bn2.momentum,
                                      m.bn2.eps)))
    return torch.cat(xs)


def _oracle_check(sd, N, R, e, r, B, nz):
    """the kernels' forward over len(e) = G * B rows against the CPU oracle: x and the running statistics bit for bit"""
    from pykg2vec_b200 import _lib
    m = au.mirror_from_state(sd, N, R, device="cuda", train=True)
    ed, rd = torch.from_numpy(np.asarray(e, np.int64)).cuda(), torch.from_numpy(np.asarray(r, np.int64)).cuda()
    nzd = [None if n is None else torch.from_numpy(np.asarray(n, np.float32)).cuda() for n in nz]
    x, _ = _lib.acre_train_fwd(m, ed, rd, B, *nzd)
    run = {}
    want = atu.oracle_fwd(sd, e, r, B, *nz, running=run)
    got = x.cpu().numpy()
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), np.abs(got - want).max()
    sdm = m.state_dict()
    for key in atu.RUNNING:
        assert np.array_equal(sdm[key].cpu().numpy().view(np.uint32), run[key].view(np.uint32)), key


@pytest.mark.parametrize("name", atu.CASES)
def test_forward_kernels_equal_oracle_bitwise_on_goldens(name):
    """the tail and head forwards of a golden case as one call of two groups, with the reference's noise: x and the
    running statistics equal the oracle's bits"""
    g = atu.load(name)
    sd = atu.state(g)
    B = len(g["h"])
    nt, nh = atu.noises(g, "tail"), atu.noises(g, "head")
    nz = [None if a is None else np.concatenate([a, b]) for a, b in zip(nt, nh)]
    _oracle_check(sd, int(g["N"]), int(g["R"]), np.concatenate([g["h"], g["t"]]), np.concatenate([g["r"], g["r"]]),
                  B, nz)


@pytest.mark.parametrize("cfg", au.FB237_CONFIGS, ids=lambda c: "%s_C%d_%s" % (c[0], c[1], "-".join(map(str, c[2]))))
def test_forward_kernels_equal_oracle_bitwise_at_fb15k237_shape(cfg):
    """N = 14,541, R = 237, two groups of B = 128 with dropout noise, at each FB15k-237 configuration"""
    N, R, B = FB237["N"], FB237["R"], 128
    sd = atu.random_state(N, R, cfg, seed=cfg[1])
    rng = np.random.RandomState(11)
    e, r = rng.randint(N, size=2 * B), rng.randint(2 * R, size=2 * B)
    e[1], r[2], e[B] = e[0], r[0], e[0]
    nz = [((rng.rand(2 * B, w) >= q) / np.float32(1 - q)).astype(np.float32)
          for w, q in ((400, 0.3), (cfg[1], 0.2), (200, 0.5))]
    _oracle_check(sd, N, R, e, r, B, nz)


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%s_C%d_%s" % (s[2], s[3], "-".join(map(str, s[4]))))
def test_forward_is_reproducible_and_per_group(shape):
    """x and the running statistics: the same bits on a repeat, and one call over two groups = two sequential calls"""
    from pykg2vec_b200 import _lib
    N, R, way, C, atrous, bias, B = shape
    e, r = _ids(N, R, 2 * B, 1)
    nz = _noise(2 * B, C)
    outs = []
    for _ in range(2):
        m = _shape_model(shape)
        x, _ = _lib.acre_train_fwd(m, e, r, B, *nz)
        outs.append((x, _running(m)))
    assert _bits_equal(outs[0][0], outs[1][0]) and all(_bits_equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))
    m = _shape_model(shape)
    parts = [_lib.acre_train_fwd(m, e[g * B:(g + 1) * B], r[g * B:(g + 1) * B], B,
                                 *[n[g * B:(g + 1) * B] for n in nz])[0] for g in range(2)]
    assert _bits_equal(torch.cat(parts), outs[0][0])
    assert all(_bits_equal(a, b) for a, b in zip(_running(m), outs[0][1]))


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "%s_C%d_%s" % (s[2], s[3], "-".join(map(str, s[4]))))
def test_forward_and_backward_match_fp64_autograd(shape):
    """two groups with dropout noise: x and the running statistics against the fp64 restatement, and every gradient
    of kge_acre_train_bwd against fp64 autograd of it.  Where bn1 has outputs within rounding of 0 (AMBIGUOUS), the
    gradients must match the restatement as it stands or with the ReLU mask of one of those outputs toggled."""
    from pykg2vec_b200 import _lib
    N, R, way, C, atrous, bias, B = shape
    Q = 2 * B
    e, r = _ids(N, R, Q, 2)
    nz = _noise(Q, C)
    m = _shape_model(shape)
    P64 = [t.detach().double().requires_grad_(True) for t in m.kge_acre_params()]
    run64 = [t.double() for t in _running(m)]
    want = _trunk64(m, P64, e, r, B, *nz, running=run64)
    params = [t.detach() for t in m.kge_acre_params()]
    x, ws = _lib.acre_train_fwd(m, e, r, B, *nz, params=params)
    assert (x.double() - want).abs().max().item() <= 2e-4 * want.abs().max().item()
    for a, b in zip(_running(m), run64):
        assert (a.double() - b).abs().max().item() <= 1e-5 * (1 + b.abs().max().item())
    up = torch.randn(Q, 200, device="cuda", generator=torch.Generator("cuda").manual_seed(7))
    grads = [torch.zeros_like(t) for t in params]
    _lib.acre_train_bwd(m, e, r, B, up, x, grads, ws, *nz, params=params)
    names = _lib.acre_train_present(m)
    amb = []
    _trunk64(m, P64, e, r, B, *nz, ambiguous=amb)
    assert len(amb) <= 32, amb
    fails = []
    for flip in [None] + amb:
        P = [t.detach().double().requires_grad_(True) for t in params]
        (_trunk64(m, P, e, r, B, *nz, flip=flip) * up.double()).sum().backward()
        scale = max(p.grad.abs().max().item() for p in P)
        bad = [name for name, got, p in zip(names, grads, P)
               if (got.double() - p.grad).abs().max().item() > 2e-3 * p.grad.abs().max().item() + 1e-5 * scale]
        if not bad:
            break
        fails.append((flip, bad))
    else:
        raise AssertionError(fails)
    assert grads[names.index("conv3_weight")].abs().max() > 0


class _Mul(torch.nn.Module):
    """a dropout module replaced by a fixed noise tensor"""

    def __init__(self, noise):
        super().__init__()
        self.noise = noise

    def forward(self, x):
        return x * self.noise


@pytest.mark.parametrize("shape", SHAPES[:2], ids=["serial", "parallel"])
def test_function_matches_torch_layers_with_the_same_noise(shape):
    """AcreTrunkFunction against _trunk_layers whose three dropout modules multiply by the same noise: x, every
    gradient, the running statistics and num_batches_tracked"""
    from pykg2vec_b200.projection import AcreTrunkFunction
    N, R, way, C, atrous, bias, B = shape
    e, r = _ids(N, R, B, 3)
    nz = _noise(B, C)
    up = torch.randn(B, 200, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
    out = []
    for kernel in (True, False):
        m = _shape_model(shape, drops=(0.3, 0.2, 0.5), kge_trunk=kernel)
        if kernel:
            x = AcreTrunkFunction.apply(m, e, r, B, *nz, *m.kge_acre_params())
            m.note_batch_stats()
        else:
            m.inp_drop = _Mul(nz[0].view(B, 1, 20, 20))
            m.feature_map_drop = _Mul(nz[1].view(B, C, 1, 1))
            m.hidden_drop = _Mul(nz[2])
            x = m._trunk_layers(e, r)
        (x * up).sum().backward()
        out.append((x.detach(), [p.grad for p in m.kge_acre_params()], m.state_dict()))
    (xa, ga, sa), (xb, gb, sb) = out
    assert (xa - xb).abs().max().item() <= 5e-5 * xb.abs().max().item()
    scale = max(g.abs().max().item() for g in gb)
    for a, b in zip(ga, gb):
        assert (a - b).abs().max().item() <= 2e-3 * b.abs().max().item() + 1e-5 * scale
    for key in sa:
        if "running" in key or "num_batches" in key:
            assert (sa[key].double() - sb[key].double()).abs().max().item() <= 1e-5, key


def _trainer(shape, opt, fused, drops=(0.0, 0.0, 0.0), lr=0.01, N=None, R=None):
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    N = N or shape[0]
    R = R or shape[1]
    m = _model(N, R, *shape[2:6], drops=drops, kge_trunk=fused)
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
    t[2] = h[0]               # one entity both a head and a tail
    hr_t, tr_h = np.zeros((B, N), np.float32), np.zeros((B, N), np.float32)
    hr_t[np.arange(B), t] = 1.0
    tr_h[np.arange(B), h] = 1.0
    hr_t[:, :3] = 1.0
    return [h, r, t, torch.from_numpy(hr_t), torch.from_numpy(tr_h)]


# in front of a training-mode BatchNorm with dropouts 0 their true gradient is ~0: the conv biases and W_gate_e.bias
# (constant per channel in front of bn1) and fc.bias (no ReLU between fc and bn2)
INVISIBLE = ("conv1.bias", "conv2.bias", "conv3.bias", "W_gate_e.bias", "fc.bias")


# (optimizer, shape): every optimizer at the two FB15k-237 defaults and the small no-bias shape; at parallel C = 32 SGD
# only, whose step is linear in the gradient (Adagrad / Adam move each element by ~lr * sign(g) on the first steps, so
# the conv weights whose gradient sits at rounding level in one arm move the other way there)
FUSED_CASES = [(opt, i) for opt in ("sgd", "adagrad", "adam") for i in (0, 1, 3)] + [("sgd", 2)]


@pytest.mark.parametrize("opt,shape", [(o, SHAPES[i]) for o, i in FUSED_CASES],
                         ids=["%s-%s" % (o, ("serial", "parallel", "parallel_c32", "parallel_nobias")[i])
                              for o, i in FUSED_CASES])
def test_fused_steps_match_autograd_on_torch_layers(opt, shape):
    """_fused_acre against train_step_projection + loss.backward() + torch.optim on _trunk_layers, dropouts 0, three
    steps.  Adagrad and Adam divide each element's step by its own gradient magnitude, so rounding noise in a near-zero
    gradient moves the element by up to lr: the bounds are those of the other training trunks' tests (SGD carries the
    comparison; under Adagrad / Adam at most 1% of the elements, and at least two (the small shape's conv banks have 45
    elements), may differ by more than 1% of lr, and the INVISIBLE parameters, whose true gradient is 0 with dropouts
    0, are held to 6 lr)."""
    N, R, B = shape[0], shape[1], shape[6]
    lr = 0.01
    a, b = _trainer(shape, opt, True, lr=lr), _trainer(shape, opt, False, lr=lr)
    assert a._acre and not b._acre and not b.model.kge_trunk
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
                assert (diff > 5 * tol).sum().item() <= max(2, 1e-2 * diff.numel()), key
    sa, sb = a.model.state_dict(), b.model.state_dict()
    for key in sa:
        if "running" in key or "num_batches" in key:
            tol = 1e-4 if (opt == "sgd" or key.startswith("bn0")) else 6 * lr
            assert (sa[key].double() - sb[key].double()).abs().max().item() <= tol, key


def test_one_row_batch_raises_before_any_launch():
    from pykg2vec_b200 import _lib
    shape = SHAPES[0]
    N = shape[0]
    m = _shape_model(shape)
    e, r = torch.tensor([5], device="cuda"), torch.tensor([1], device="cuda")
    before = (_lib.launch_count(), _running(m))
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        m(e, r)
    with pytest.raises(ValueError, match="Expected more than 1 value per channel when training"):
        _trainer(shape, "adam", True).train_batch_device([e, r, e, torch.zeros(1, N, device="cuda"),
                                                          torch.zeros(1, N, device="cuda")])
    assert _lib.launch_count() == before[0]
    assert all(torch.equal(a, b) for a, b in zip(before[1], _running(m)))


@pytest.mark.parametrize("shape", SHAPES[:2], ids=["serial", "parallel"])
def test_fused_steps_with_dropout_learn_and_repeat(shape):
    N, R = shape[0], shape[1]
    batch = _batch(N, R, 32, 9)
    runs = []
    for rep in range(2):
        tr = _trainer(shape, "adam", True, drops=(0.3, 0.2, 0.5), lr=0.01)
        torch.manual_seed(42)
        runs.append([tr.train_batch(batch) for _ in range(30)])
    assert np.isfinite(runs[0]).all() and np.mean(runs[0][-5:]) < np.mean(runs[0][:5])
    # the three dropouts follow torch.manual_seed: a reseeded run repeats up to the order of the float atomics
    assert np.allclose(runs[0][:3], runs[1][:3], rtol=1e-5, atol=0)
    tr = _trainer(shape, "adam", True, drops=(0.3, 0.2, 0.5), lr=0.01)
    torch.manual_seed(43)
    assert abs(tr.train_batch(batch) - runs[0][0]) > 1e-6 * runs[0][0]


def test_evaluator_after_fused_training_matches_the_torch_path():
    """after fused adam steps, the Evaluator's raw ranks (kge_acre_trunk_fwd + kge_proj_rank) against ranks counted
    from the torch layers' predictions (eval mode) on the same weights"""
    from pykg2vec_b200.evaluator import Evaluator
    shape = SHAPES[0]
    N, R, B = shape[0], shape[1], shape[6]
    tr = _trainer(shape, "adam", True, lr=0.003)
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


def _fb237_trainer(cfg, fused):
    way, C, atrous, bias = cfg
    return _trainer((0, 0, way, C, atrous, bias, 128), "adam", fused, drops=(0.3, 0.2, 0.5), lr=0.0001,
                    N=FB237["N"], R=FB237["R"])


def _fb237_batch(tr, B=128):
    batch = _batch(FB237["N"], FB237["R"], B, 3)
    return tr._projection_batch(batch)[0]


@pytest.mark.parametrize("cfg", au.FB237_CONFIGS, ids=lambda c: "%s_C%d" % (c[0], c[1]))
def test_fused_step_peak_memory_at_the_bench_shape(cfg):
    """one fused step at the FB15k-237 shape (B = 128, Adam) allocates at most the trunk's workspace for 2B rows +
    32 MB above the standing tensors: the [2B, N] predictions and one [B, N] gradient (22 MB), the noise and x / gx"""
    from pykg2vec_b200 import _lib
    tr = _fb237_trainer(cfg, True)
    ids = _fb237_batch(tr)
    tr.train_batch_device(ids)   # warm-up: the optimizer state and scratch exist from build_model on
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    tr.train_batch_device(ids)
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    ws = _lib.acre_train_workspace_bytes(tr.model, 256, 128)
    assert 0 < ws and peak <= ws + (32 << 20), (peak, ws)


@pytest.mark.parametrize("cfg", au.FB237_CONFIGS[:2], ids=["serial", "parallel"])
def test_training_steps_run_no_cudnn_convolution(cfg):
    """AcrE(...).train() with CUDA tables: neither the fused step nor loss.backward() through AcreTrunkFunction
    launches a cuDNN / convolution kernel"""
    from torch.profiler import ProfilerActivity, profile
    for fused in (True, False):
        tr = _fb237_trainer(cfg, True)
        if not fused:
            tr._acre = False   # the autograd path on the kernels: train_step_projection + loss.backward()
        ids = _fb237_batch(tr)
        tr.train_batch_device(ids)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            tr.train_batch_device(ids)
            torch.cuda.synchronize()
        names = [ev.name for ev in prof.events() if ev.device_type == torch.autograd.DeviceType.CUDA]
        assert any("acre_tr_" in n for n in names), names[:20]
        cudnn = ("cudnn", "xmma", "implicit_gemm", "conv2d", "convolution", "depthwise", "winograd", "fprop", "dgrad",
                 "wgrad")
        bad = [n for n in names if any(w in n.lower() for w in cudnn)]
        assert not bad, (fused, bad[:10])
