"""TuckER's kernels on the device (kge_tucker_* of include/kge_b200.h) and every layer above them: the kernels against
the CPU oracle (tests/oracle_tucker) bit for bit, the model against the reference's outputs (tests/golden/tucker/),
the autograd Function against the torch layers fed the same noise, the Trainer's fused step against
loss.backward() + torch.optim on the torch layers, the Evaluator's per-call core matrices, the memory bound that
rules out a per-sample matrix, and the unmodified reference Trainer driving the class."""
import types

import numpy as np
import pytest
import torch

import dropin_util as du
import golden_util as gu
import tucker_util as tu

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _evaluator(m, N):
    from pykg2vec_b200.evaluator import Evaluator
    ev = object.__new__(Evaluator)
    ev.model, ev.config = m, types.SimpleNamespace(device="cuda", tot_entity=N)
    ev._filter_cache, ev._workspace = {}, None
    return ev


@pytest.mark.parametrize("name", tu.CASES)
def test_kernels_equal_oracle_bitwise_and_model_matches_reference(name):
    from pykg2vec_b200 import _lib
    g = tu.load(name)
    tabs = tu.tables(g)
    dtabs = [_cuda(t) for t in tabs]
    ids, slot = tu.slots(g["r"])
    want_M = tu.oracle_cores(tabs, ids)
    M = _lib.tucker_cores(dtabs, _cuda(ids))
    assert _bits_equal(M.cpu().numpy(), want_M)
    nz = tu.noises(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        n0, n1, n2 = nz[tag] if nz else (None, None, None)
        got = _lib.tucker_trunk_fwd(dtabs, M, _cuda(e), _cuda(slot), noise0=_cuda(n0) if nz else None,
                                    noise1=_cuda(n1) if nz else None, noise2=_cuda(n2) if nz else None, save=True)
        want = tu.oracle_trunk(tabs, want_M, e, slot, n0, ("explicit", n1) if nz else None, n2)
        for a, b in zip(got, want):
            assert _bits_equal(a.cpu().numpy(), b)
    m = tu.mirror(g).eval()
    h, r, t = _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])
    with torch.no_grad():
        assert gu.rel_err(m(h, r, direction="tail").cpu().numpy(), g["preds_tail"]).max() < 1e-4
        assert gu.rel_err(m(t, r, direction="head").cpu().numpy(), g["preds_head"]).max() < 1e-4
        # the kernel path and the torch layers are the same function
        m.kge_trunk = False
        ref = m.proj_query(h, r)
        m.kge_trunk = True
        assert (m.proj_query(h, r) - ref).abs().max().item() < 1e-5


@pytest.mark.parametrize("name", tu.CASES)
def test_evaluator_ranks_with_per_call_cores(name, monkeypatch):
    """ranks equal the reference's, filtered and raw, with the matrices built once and reused over several query
    batches and both directions, and again with a budget that holds one matrix at a time"""
    from pykg2vec_b200 import projection
    g = tu.load(name)
    m = tu.mirror(g).eval()
    rows = g["query_rows"]
    hs, rs, ts = g["h"][rows], g["r"][rows], g["t"][rows]
    ev = _evaluator(m, int(g["N"]))
    ev.QUERY_BATCH = 4
    made = []
    real = projection.TuckerCores

    def counting(*a, **k):
        made.append(real(*a, **k))
        return made[-1]
    monkeypatch.setattr(projection, "TuckerCores", counting)
    with torch.no_grad():
        got = ev.rank_triples(hs, rs, ts, (g["filt_t_ptr"], g["filt_t_idx"]), (g["filt_h_ptr"], g["filt_h_idx"]))
        assert len(made) == 1 and made[0].builds == 1 and len(rows) > 2 * ev.QUERY_BATCH
        raw = ev.rank_triples(hs, rs, ts)
        m.CORES_BUDGET = 4 * int(g["d1"]) ** 2          # one matrix per chunk
        small = ev.rank_triples(hs, rs, ts, (g["filt_t_ptr"], g["filt_t_idx"]), (g["filt_h_ptr"], g["filt_h_idx"]))
        assert made[-1].per == 1 and made[-1].builds > 1
        x_small = m.proj_query(_cuda(hs), _cuda(rs))
        m.CORES_BUDGET = type(m).CORES_BUDGET
        assert torch.equal(x_small, m.proj_query(_cuda(hs), _cuda(rs)))
    assert np.array_equal(got, g["ranks"]) and np.array_equal(small, g["ranks"])
    assert np.array_equal(raw[:, [0, 2]], g["ranks"][:, [0, 2]]) and np.array_equal(raw[:, 0], raw[:, 1])


def _step_autograd(m, g, smoothing):
    from pykg2vec_b200.trainer import Trainer
    tr = object.__new__(Trainer)
    tr.model = m
    tr.config = types.SimpleNamespace(device="cuda", label_smoothing=smoothing, tot_entity=int(g["N"]))
    m.zero_grad()
    loss = tr.train_step_projection(_cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"]), _cuda(g["lab_tail"]),
                                    _cuda(g["lab_head"]))
    loss.backward()
    return loss.item(), [p.weight.grad.cpu().numpy() for p in m.parameter_list]


@pytest.mark.parametrize("name", ["tucker_d200", "tucker_33x7"])
def test_autograd_function_matches_reference_gradients(name):
    g = tu.load(name)
    m = tu.mirror(g).train()
    loss, grads = _step_autograd(m, g, float(g["label_smoothing"]))
    assert abs(loss - float(g["loss"])) <= 1e-5 * abs(float(g["loss"]))
    tu.golden_grad_check(g, grads, 5e-4)


def test_autograd_function_matches_torch_layers_with_the_same_noise():
    """explicit mask mode against the reference's per-sample formulation in torch, fed the reference's captured noise"""
    from pykg2vec_b200.projection import TuckerTrunkFunction
    g = tu.load("tucker_50x30_drop")
    nz = tu.noises(g)
    e, r = _cuda(g["h"]), _cuda(g["r"])
    n0, n1, n2 = [_cuda(a) for a in nz["tail"]]
    up = torch.randn(len(g["h"]), int(g["d1"]), device="cuda", generator=torch.Generator("cuda").manual_seed(3))
    out = []
    for kernel in (True, False):
        m = tu.mirror(g, drops=(0, 0, 0))
        ent, rel, W = m.kge_tucker_tables()
        if kernel:
            x = TuckerTrunkFunction.apply(e, r, n0, ("explicit", n1), n2, ent, rel, W)
        else:
            eh = torch.nn.functional.normalize(ent[e], p=2, dim=1) * n0
            Wm = torch.matmul(rel[r], W).view(-1, m.d1, m.d1) * n1
            x = torch.nn.functional.normalize(torch.matmul(eh.view(-1, 1, m.d1), Wm).view(-1, m.d1), p=2, dim=1) * n2
        (x * up).sum().backward()
        out.append([x.detach()] + [w.grad for w in (ent, rel, W)])
    for a, b in zip(*out):
        assert (a - b).abs().max().item() <= 2e-5 * b.abs().max().item()


def _trainer(g, opt, fused, drops=None, lr=0.01):
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    m = tu.mirror(g, drops=drops, kge_trunk=fused)
    cfg = types.SimpleNamespace(device="cuda", optimizer=opt, learning_rate=lr, fused_step=fused,
                                label_smoothing=0.1, tot_entity=int(g["N"]), batch_size=len(g["h"]),
                                knowledge_graph=None)
    tr = Trainer(m, cfg)
    ev = trmod.Evaluator
    trmod.Evaluator = lambda *a, **k: None     # no evaluation here: the config carries no knowledge graph
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev
    return tr


@pytest.mark.parametrize("opt", ["sgd", "adagrad", "adam"])
def test_fused_steps_match_autograd_on_torch_layers(opt):
    """_fused_tucker against train_step_projection + loss.backward() + torch.optim on _trunk_layers, dropouts 0
    (tolerances of the equivalent ProjE test)"""
    g = tu.load("tucker_33x7")
    a, b = _trainer(g, opt, True, (0, 0, 0)), _trainer(g, opt, False, (0, 0, 0))
    assert a._tucker and not b._tucker and not b.model.kge_trunk
    batch = [g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"]]
    for step in range(3):
        la, lb = a.train_batch(batch), b.train_batch(batch)
        assert abs(la - lb) <= 1e-5 * abs(lb)
    for key, pa, pb in zip(tu.KEYS, a.model.parameter_list, b.model.parameter_list):
        wa, wb = pa.weight.detach(), pb.weight.detach()
        assert (wa - wb).abs().max().item() <= 2e-3 * 0.01 + 1e-5 * wb.abs().max().item(), key


def test_fused_steps_with_dropout_learn_and_repeat():
    g = tu.load("tucker_50x30_drop")
    batch = [g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"]]
    runs = []
    for rep in range(2):
        tr = _trainer(g, "adam", True, lr=0.02)
        torch.manual_seed(42)
        runs.append([tr.train_batch(batch) for _ in range(30)])
    assert np.isfinite(runs[0]).all() and np.mean(runs[0][-5:]) < np.mean(runs[0][:5])
    # the three dropouts follow torch.manual_seed: a reseeded run repeats up to the order of the float atomics
    # (loss and gradient sums), another seed draws other masks
    assert np.allclose(runs[0][:3], runs[1][:3], rtol=1e-5, atol=0)
    tr = _trainer(g, "adam", True, lr=0.02)
    torch.manual_seed(43)
    assert abs(tr.train_batch(batch) - runs[0][0]) > 1e-4 * runs[0][0]


def test_counter_mask_on_device_equals_oracle():
    from pykg2vec_b200 import _lib
    m = _lib.tucker_mask1(2 ** 40 + 17, 2 ** 33 + 3, 0.4, 5, 21).cpu().numpy()
    assert _bits_equal(m, tu.oracle_mask1(2 ** 40 + 17, 2 ** 33 + 3, 0.4, 5, 21))


def test_fused_step_never_holds_a_per_sample_matrix():
    """FB15k-237 widths (d1 = d2 = 200, B = 128, R = 237): the step's peak above the standing allocations and the
    [B, N] tail buffers (predictions and their gradient, both directions, and the float label rows) stays below
    B * d1 * d1 * 4 bytes, the size of ONE per-sample matrix batch"""
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    N, R, d, B = 14541, 237, 200, 128
    torch.manual_seed(0)
    m = import_model("tucker")(tot_entity=N, tot_relation=R, ent_hidden_size=d, rel_hidden_size=d, lmbda=0.0,
                               input_dropout=0.3, hidden_dropout1=0.4, hidden_dropout2=0.5).cuda()
    cfg = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=1e-3, fused_step=True,
                                label_smoothing=0.1, tot_entity=N, batch_size=B, knowledge_graph=None)
    tr = Trainer(m, cfg)
    ev, trmod.Evaluator = trmod.Evaluator, (lambda *a, **k: None)
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev
    gen = torch.Generator("cuda").manual_seed(1)
    ids = [torch.randint(N, (B,), device="cuda", generator=gen), torch.randint(R, (B,), device="cuda", generator=gen),
           torch.randint(N, (B,), device="cuda", generator=gen)]
    labels = [(torch.rand(B, N, device="cuda", generator=gen) < 0.001).float() for _ in range(2)]
    for _ in range(2):
        tr.train_batch_device(ids + labels)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    tr.train_batch_device(ids + labels)
    torch.cuda.synchronize()
    extra = torch.cuda.max_memory_allocated() - base
    tail = 4 * B * N * 4        # preds [2B, N] and one direction's gradient at a time [B, N], rounded up to two
    assert extra - tail < B * d * d * 4, (extra, tail)


def test_unsupported_width_uses_the_torch_layers():
    from pykg2vec_b200 import _lib, import_model
    m = import_model("tucker")(tot_entity=20, tot_relation=3, ent_hidden_size=260, rel_hidden_size=4, lmbda=0.0,
                               input_dropout=0.0, hidden_dropout1=0.0, hidden_dropout2=0.0).cuda().eval()
    e, r = torch.tensor([1, 5], device="cuda"), torch.tensor([2, 0], device="cuda")
    with pytest.raises(_lib.KgeNotSupported):
        _lib.tucker_cores(m.kge_tucker_tables(), r)
    with torch.no_grad():
        assert m.proj_query_cores(r) is None
        assert torch.equal(m.proj_query(e, r), m._trunk_layers(e, r))
    m.train()
    m(e, r).sum().backward()
    assert m.W.weight.grad is not None


DROPIN_FLOW = r"""
import json, os, sys
import numpy as np
import torch
import dropin_util as du
B200Importer = du.b200_importer_class()
ds = du.write_dataset(os.path.abspath("data"))
argv = ["-mn", "tucker", "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1", "-ds", "syn", "-dsp", ds,
        "-device", "cuda", "-km", "32", "-kr", "16"]
tr = du.run_cli_flow(argv, B200Importer)
out = {"cls": type(tr.model).__module__ + "." + type(tr.model).__name__, "cuda": next(tr.model.parameters()).is_cuda,
       "kernels": bool(tr.model.kge_trunk),
       "losses": [float(v) for _, v in tr.training_results],
       "mr_finite": all(bool(np.isfinite(v)) for v in tr.evaluator.metric_calculator.mr.values()),
       "infer": [len(tr.infer_tails(1, 10, topk=5)), len(tr.infer_heads(10, 20, topk=5))]}
print("RESULT " + json.dumps(out))
"""


@pytest.mark.skipif(not du.reference_available(), reason="oracle/_ref not installed (no reference checkout at build())")
def test_reference_trainer_drives_tucker(tmp_path):
    """the unmodified reference CLI flow (Importer -> Trainer.build_model / train_model with its mini_test ->
    Evaluator -> infer_*) with this package's TuckER patched into Importer, -device cuda: loss.backward() and
    torch.optim train through the kernels"""
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
    assert out["cls"] == "pykg2vec_b200.projection.TuckER" and out["cuda"] and out["kernels"]
    assert len(out["losses"]) == 2 and np.isfinite(out["losses"]).all()
    assert out["losses"][1] < out["losses"][0]
    assert out["mr_finite"] and out["infer"] == [5, 5]
