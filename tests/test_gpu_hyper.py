"""-m gpu tests of HypER (pykg2vec/models/projection.py:508-618): the inference-trunk kernels
(kge_hyper_trunk_fwd) vs the CPU oracle bit for bit, and the mirror class vs the golden vectors the
reference itself produced (tests/golden/make_golden_hyper.py): eval predictions, Evaluator ranks, the
training step's loss / gradients / BatchNorm statistics, a device-Generator epoch and the unmodified
reference Trainer driving the class."""
import ctypes
import types

import numpy as np
import pytest
import torch

import dropin_util as du
import golden_util as gu
import gpu_util as gpu
import hyper_util as hu
import oracle

pytestmark = pytest.mark.gpu
FB237 = dict(N=14541, R=237, de=200, dr=200)


def _L():
    from pykg2vec_b200 import _lib
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _fb237_mirror(seed=237):
    """a HypER at the FB15k-237 shape with seeded parameters and non-trivial BN buffers, eval mode"""
    from pykg2vec_b200 import import_model
    st = hu.random_state(FB237["N"], FB237["R"], FB237["de"], FB237["dr"], seed)
    m = import_model("hyper")(tot_entity=FB237["N"], tot_relation=FB237["R"], ent_hidden_size=FB237["de"],
                              rel_hidden_size=FB237["dr"], input_dropout=0.2, hidden_dropout=0.3,
                              feature_map_dropout=0.2, device="cuda")
    m.load_state_dict({k: torch.from_numpy(v) for k, v in st.items()}, strict=True)
    return st, m.cuda().eval()


# ---- trunk kernels vs the oracle ----------------------------------------------------------------
@pytest.mark.parametrize("name", hu.CASES)
def test_trunk_kernel_bit_exact_vs_oracle_on_goldens(name):
    L = _L()
    g = hu.load(name)
    m = hu.mirror(g)
    st = hu.state(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        got = L.hyper_trunk_fwd(m, _cuda(e), _cuda(g["r"])).cpu().numpy()
        assert np.array_equal(gpu.bits(got), gpu.bits(hu.oracle_trunk_fwd(st, e, g["r"])))
        assert np.abs(got - g["x_" + tag]).max() <= 1e-5


@pytest.mark.parametrize("Q", [1, 77, 512])
def test_trunk_kernel_bit_exact_vs_oracle_at_fb15k237_shape(Q):
    L = _L()
    st, m = _fb237_mirror()
    rng = np.random.RandomState(Q)
    e, r = rng.randint(FB237["N"], size=Q), rng.randint(FB237["R"], size=Q)
    e[0], r[-1] = 0, 0
    got = L.hyper_trunk_fwd(m, _cuda(e), _cuda(r)).cpu().numpy()
    want = hu.oracle_trunk_fwd(st, e, r)
    assert np.array_equal(gpu.bits(got), gpu.bits(want))
    assert (got > 0).any()


def test_trunk_argument_errors():
    """de < 9 has no convolution output: KGE_ENOTSUP; a short workspace: KGE_EWORKSPACE, nothing written;
    Q = 0 is a no-op"""
    L = _L()
    from pykg2vec_b200 import import_model
    small = import_model("hyper")(tot_entity=20, tot_relation=3, ent_hidden_size=8, rel_hidden_size=4, input_dropout=0.0,
                                  hidden_dropout=0.0, feature_map_dropout=0.0, device="cuda").cuda().eval()
    ids = torch.zeros(2, dtype=torch.int64, device="cuda")
    with pytest.raises(L.KgeNotSupported):
        L.hyper_trunk_fwd(small, ids, ids)
    g = hu.load(hu.CASES[0])
    m = hu.mirror(g)
    assert L.hyper_trunk_fwd(m, ids[:0], ids[:0]).shape == (0, int(g["ent_hidden_size"]))
    p = L.KgeHyper()
    p.ent_hidden_size, p.rel_hidden_size, p.num_rel = int(g["ent_hidden_size"]), int(g["rel_hidden_size"]), int(g["R"])
    p.bn0_eps = p.bn1_eps = p.bn2_eps = 1e-5
    keep = {n: t.detach() for n, t in (("ent", m.ent_embeddings.weight), ("rel", m.rel_embeddings.weight),
                                       ("fc1_weight", m.fc1.weight), ("fc1_bias", m.fc1.bias),
                                       ("fc_weight", m.fc.weight), ("fc_bias", m.fc.bias))}
    for bn in ("bn0", "bn1", "bn2"):
        mod = getattr(m, bn)
        keep.update({bn + "_weight": mod.weight.detach(), bn + "_bias": mod.bias.detach(),
                     bn + "_mean": mod.running_mean, bn + "_var": mod.running_var})
    for n in L.HYPER_FIELDS:
        setattr(p, n, keep[n].data_ptr())
    need = int(L.lib().kge_hyper_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(2)))
    assert need > 0
    ws = torch.empty(need - 4, dtype=torch.uint8, device="cuda")
    x = torch.full((2, p.ent_hidden_size), 7.0, device="cuda")
    rc = L.lib().kge_hyper_trunk_fwd(ctypes.byref(p), L._ptr(ids), L._ptr(ids), ctypes.c_int64(2), L._ptr(x), L._ptr(ws),
                                     ctypes.c_int64(ws.numel()), L._stream())
    assert rc == -4 and (x == 7.0).all()


# ---- the mirror vs the reference's outputs --------------------------------------------------------
@pytest.mark.parametrize("name", hu.CASES)
def test_eval_forward_matches_reference(name):
    """model.forward(e, r, direction) in eval mode vs the reference's output: <= 1e-4 relative"""
    g = hu.load(name)
    m = hu.mirror(g)
    h, r, t = _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])
    with torch.no_grad():
        pt = m(h, r, direction="tail").cpu().numpy()
        ph = m(t, r, direction="head").cpu().numpy()
        xt = m.proj_query(h, r, "tail").cpu().numpy()
    assert gu.rel_err(pt, g["preds_tail"]).max() <= 1e-4 and gu.rel_err(ph, g["preds_head"]).max() <= 1e-4
    assert np.abs(xt - g["x_tail"]).max() <= 1e-5
    # grad-enabled eval forward runs the torch layers: same predictions
    pt2 = m(h, r, direction="tail").detach().cpu().numpy()
    assert gu.rel_err(pt2, g["preds_tail"]).max() <= 1e-4
    with torch.no_grad():
        rank = m.predict_tail_rank(h[:1], r[:1], topk=int(g["N"])).cpu().numpy()[0]
    assert rank[-1] == int(np.argmax(pt[0])) and rank[0] == int(np.argmin(pt[0]))


def _evaluator(m, N):
    from pykg2vec_b200.evaluator import Evaluator
    ev = object.__new__(Evaluator)
    ev.model, ev.config = m, types.SimpleNamespace(device="cuda", tot_entity=N)
    ev._filter_cache, ev._workspace = {}, None
    return ev


@pytest.mark.parametrize("name", hu.CASES)
def test_evaluator_ranks_match_reference(name):
    g = hu.load(name)
    m = hu.mirror(g)
    Q = g["ranks"].shape[0]
    ev = _evaluator(m, int(g["N"]))
    with torch.no_grad():
        got = ev.rank_triples(g["h"][:Q], g["r"][:Q], g["t"][:Q], (g["filt_t_ptr"], g["filt_t_idx"]),
                              (g["filt_h_ptr"], g["filt_h_idx"]))
        assert ev.last_d2h_bytes == 16 * Q
        raw = ev.rank_triples(g["h"][:Q], g["r"][:Q], g["t"][:Q])
        assert ev.last_d2h_bytes == 16 * Q
    assert np.array_equal(got, g["ranks"])
    assert np.array_equal(raw[:, 0], g["ranks"][:, 0]) and np.array_equal(raw[:, 2], g["ranks"][:, 2])
    assert np.array_equal(raw[:, 1], raw[:, 0]) and np.array_equal(raw[:, 3], raw[:, 2])


def test_evaluator_ranks_at_fb15k237_shape_match_oracle():
    """Evaluator.rank_triples (kernel trunk + kge_proj_rank) == the oracle's trunk + rank counts on sampled
    queries at N = 14,541, R = 237, d = 200, with filters"""
    st, m = _fb237_mirror(seed=5)
    N, R = FB237["N"], FB237["R"]
    rng = np.random.RandomState(11)
    Q = 96
    h, r, t = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    (ft, fh) = gpu.random_filters_csr(rng, N, h, r, t, per_query=30)
    ev = _evaluator(m, N)
    with torch.no_grad():
        got = ev.rank_triples(h, r, t, ft, fh)
    assert ev.last_d2h_bytes == 16 * Q
    E, b = st["ent_embeddings.weight"], st["b"]
    want = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(hu.oracle_trunk_fwd(st, h, r), E, b, t, ft, 0, want)
    oracle.proj_rank(hu.oracle_trunk_fwd(st, t, r), E, b, h, fh, 1, want)
    assert np.array_equal(got, want)
    assert (got[:, 1] <= got[:, 0]).all() and (got[:, 3] <= got[:, 2]).all()


@pytest.mark.parametrize("name", hu.CASES)
def test_training_step_matches_reference_autograd(name):
    """train_step_projection (trainer.py:159-174): loss and the gradient of every parameter vs the
    reference's own backward (fc1's gradient arrives through the per-query filters); BatchNorm running
    statistics after the two forwards."""
    from pykg2vec_b200.trainer import Trainer
    g = hu.load(name)
    m = hu.mirror(g, train=True)
    tr = object.__new__(Trainer)
    tr.model = m
    tr.config = types.SimpleNamespace(device="cuda", label_smoothing=float(g["label_smoothing"]), tot_entity=int(g["N"]))
    m.zero_grad()
    loss = tr.train_step_projection(_cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"]), _cuda(g["tr_labels_tail"]),
                                    _cuda(g["tr_labels_head"]))
    loss.backward()
    assert abs(loss.item() - float(g["tr_loss"])) <= 1e-5 * abs(float(g["tr_loss"]))
    seen = set()
    for key, p in m.named_parameters():
        got, want = p.grad.detach().cpu().numpy(), g["grad_" + key]
        # bn0 / fc biases in front of a training-mode BatchNorm have a true gradient of 0: relative bound + floor
        assert np.abs(got - want).max() <= 5e-4 * np.abs(want).max() + 1e-7, key
        seen.add(key)
    assert seen == {k[5:] for k in g if k.startswith("grad_")}
    assert not m.rel_embeddings.weight.grad[0].any()          # padding_idx=0, relation 0 is in the batch
    assert m.ent_embeddings.weight.grad[0].any()              # entity row 0 still gets the tail product's gradient
    for key, v in m.state_dict().items():
        if "running" in key:
            assert np.abs(v.cpu().numpy() - g["sd_after_" + key]).max() < 1e-5, key


def test_epoch_on_device_generator():
    """Generator (device label rows) -> Trainer.train_model_epoch -> batched Evaluator, HypER, adam"""
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.generator import Generator
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    from pykg2vec_b200.trainer import Trainer
    kg = SyntheticKnowledgeGraph(200, 5, 2000, 60, 60, seed=3)
    cfg = SyntheticConfig(kg, device="cuda", optimizer="adam", learning_rate=0.003, batch_size=64, neg_rate=0,
                          ent_hidden_size=48, rel_hidden_size=32, input_dropout=0.0, feature_map_dropout=0.0,
                          hidden_dropout=0.0, label_smoothing=0.1, test_num=50)
    torch.manual_seed(0)
    model = import_model("hyper")(**cfg.__dict__)
    tr = Trainer(model, cfg)
    tr.build_model()
    gen = Generator(model, cfg, seed=1)
    losses = [tr.train_model_epoch(gen, num_batch=10) for _ in range(4)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
    model.eval()
    scores = tr.evaluator.mini_test(epoch=0)
    assert set(scores) == {"mr", "fmr", "mrr", "fmrr"} and 1.0 <= scores["fmr"] <= scores["mr"] <= 200.0


# The reference's Generator forks its worker processes; a fork taken after this test process has run OpenMP
# regions (the oracle) can deadlock the child, so the reference's flow runs in a fresh interpreter.
DROPIN_FLOW = r"""
import json, os, sys
import numpy as np
import torch
import dropin_util as du
B200Importer = du.b200_importer_class()
ds = du.write_dataset(os.path.abspath("data"))
argv = ["-mn", "hyper", "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1", "-ds", "syn", "-dsp", ds,
        "-device", "cuda", "-km", "32", "-kr", "32"]
tr = du.run_cli_flow(argv, B200Importer)
out = {"cls": type(tr.model).__module__ + "." + type(tr.model).__name__, "cuda": next(tr.model.parameters()).is_cuda,
       "losses": [float(v) for _, v in tr.training_results],
       "mr_finite": all(bool(np.isfinite(v)) for v in tr.evaluator.metric_calculator.mr.values()),
       "infer": [len(tr.infer_tails(1, 10, topk=5)), len(tr.infer_heads(10, 20, topk=5))]}
# the reference's per-query ranks over this package's forward == the batched rank path on the same weights
from pykg2vec_b200.evaluator import Evaluator as B200Evaluator
ev = B200Evaluator(tr.model, tr.config)
tr.model.eval()
ev.full_test(epoch=0)
with torch.no_grad():
    tr.evaluator.full_test(0)
ref_mc = tr.evaluator.metric_calculator
got = np.stack([ev.metric_calculator.rank_tail, ev.metric_calculator.rank_head], axis=1)
want = np.stack([ref_mc.rank_tail, ref_mc.rank_head], axis=1)
out["rank_mismatch"] = float((got != want).mean())
print("RESULT " + json.dumps(out))
"""


@pytest.mark.skipif(not du.reference_available(), reason="oracle/_ref not installed (no reference checkout at build())")
def test_reference_trainer_drives_hyper(tmp_path):
    """the unmodified reference CLI flow (Importer -> Trainer.build_model / train_model -> Evaluator -> infer_*)
    with this package's HypER patched into Importer, -device cuda"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", DROPIN_FLOW], cwd=str(tmp_path), env=env, capture_output=True,
                         text=True, timeout=300)
    lines = [l for l in res.stdout.splitlines() if l.startswith("RESULT ")]
    assert res.returncode == 0 and lines, res.stderr[-4000:]
    out = json.loads(lines[-1][len("RESULT "):])
    assert out["cls"] == "pykg2vec_b200.projection.HypER" and out["cuda"]
    assert len(out["losses"]) == 2 and np.isfinite(out["losses"]).all()
    assert out["losses"][1] < out["losses"][0]          # the loss goes down between the two epochs
    assert out["mr_finite"] and out["infer"] == [5, 5]
    assert out["rank_mismatch"] < 0.02, out["rank_mismatch"]   # only exact ties may order differently under topk
