"""-m gpu tests of AcrE (pykg2vec/models/projection.py:621-746): the inference-trunk kernels (kge_acre_trunk_fwd)
vs the CPU oracle bit for bit, and the mirror class vs the golden vectors the reference itself produced
(tests/golden/make_golden_acre.py): eval predictions, Evaluator ranks, the training step's loss / gradients /
BatchNorm statistics, a device-Generator epoch and the unmodified reference Trainer driving the class."""
import ctypes
import types

import numpy as np
import pytest
import torch

import acre_util as au
import dropin_util as du
import golden_util as gu
import gpu_util as gpu
import oracle

pytestmark = pytest.mark.gpu
FB237 = dict(N=14541, R=237)


def _L():
    from pykg2vec_b200 import _lib
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cfg_id(c):
    return "%s_C%d_%d%d%d_%s" % (c[0], c[1], *c[2], "bias" if c[3] else "nobias")


# ---- trunk kernels vs the oracle ----------------------------------------------------------------
@pytest.mark.parametrize("name", au.CASES)
def test_trunk_kernel_bit_exact_vs_oracle_on_goldens(name):
    L = _L()
    g = au.load(name)
    m = au.mirror(g).eval()
    st = au.state(g)
    for tag, e in (("tail", g["h"]), ("head", g["t"])):
        got = L.acre_trunk_fwd(m, _cuda(e), _cuda(g["r"])).cpu().numpy()
        assert np.array_equal(gpu.bits(got), gpu.bits(au.oracle_trunk_fwd(st, e, g["r"])))
        assert np.abs(got - g["x_" + tag]).max() <= 1e-5


@pytest.fixture(scope="module")
def fb237_models():
    """one AcrE per configuration at N = 14,541, R = 237: (state, eval-mode mirror)"""
    out = {}
    for i, cfg in enumerate(au.FB237_CONFIGS):
        st = au.random_state(FB237["N"], FB237["R"], cfg, seed=237 + i)
        out[cfg] = (st, au.mirror_from_state(st, FB237["N"], FB237["R"], dropout=0.3).eval())
    return out


@pytest.mark.parametrize("cfg", au.FB237_CONFIGS, ids=_cfg_id)
@pytest.mark.parametrize("Q", [1, 77, 512])
def test_trunk_kernel_bit_exact_vs_oracle_at_fb15k237_shape(fb237_models, cfg, Q):
    L = _L()
    st, m = fb237_models[cfg]
    rng = np.random.RandomState(Q)
    e, r = rng.randint(FB237["N"], size=Q), rng.randint(FB237["R"], size=Q)
    e[0], r[-1] = 0, 0
    got = L.acre_trunk_fwd(m, _cuda(e), _cuda(r)).cpu().numpy()
    want = au.oracle_trunk_fwd(st, e, r)
    assert np.array_equal(gpu.bits(got), gpu.bits(want))
    assert (got > 0).any()


@pytest.mark.parametrize("cfg", [au.FB237_CONFIGS[0], au.FB237_CONFIGS[2]], ids=_cfg_id)
def test_chunked_calls_equal_one_call(fb237_models, cfg):
    """queries are independent: a cap that splits Q = 77 into chunks of 10 (and of 1) gives the same bits"""
    L = _L()
    st, m = fb237_models[cfg]
    way, C, atrous, _ = cfg
    per_query = L.acre_trunk_workspace_bytes(way, C, atrous, 200, 2 * FB237["R"], 1)
    rng = np.random.RandomState(3)
    e, r = _cuda(rng.randint(FB237["N"], size=77)), _cuda(rng.randint(FB237["R"], size=77))
    whole = L.acre_trunk_fwd(m, e, r, cap=per_query * 77)
    for cap in (per_query * 10, per_query, 1):
        assert torch.equal(L.acre_trunk_fwd(m, e, r, cap=cap).view(torch.int32), whole.view(torch.int32))
    # the default cap splits an Evaluator-sized batch
    assert per_query * 8192 > L.ACRE_WORKSPACE_CAP


def _struct_for(L, m):
    p = L.acre_struct(m.way, m.in_channels, (m.first_atrous, m.second_atrous, m.third_atrous), m.hidden_size,
                      m.rel_embeddings.weight.shape[0])
    p.bn0_eps = p.bn1_eps = p.bn2_eps = 1e-5
    sd = m.state_dict()
    keep = {f: sd[k] for f, k in au.KEYS.items() if k in sd}
    for f, t in keep.items():
        setattr(p, f, t.data_ptr())
    return p, keep


def test_trunk_argument_errors_on_device():
    """hidden_size != 200 and a serial C over the shared-memory bound: KGE_ENOTSUP (KgeNotSupported from the
    eval path); a short workspace: KGE_EWORKSPACE, nothing written; Q = 0 is a no-op that accepts null ids and
    output"""
    L = _L()
    from pykg2vec_b200 import import_model
    ids = torch.zeros(2, dtype=torch.int64, device="cuda")
    for kw in (au.kwargs("serial", 4, (1, 2, 2), True, 20, 3, hidden_size=100),
               au.kwargs("serial", 47, (1, 2, 2), True, 20, 3)):
        bad = import_model("acre")(**kw).cuda().eval()
        with pytest.raises(L.KgeNotSupported):
            L.acre_trunk_fwd(bad, ids, ids)
        with torch.no_grad(), pytest.raises(L.KgeNotSupported):
            bad(ids, ids)
    for name in au.CASES:
        g = au.load(name)
        m = au.mirror(g).eval()
        assert L.acre_trunk_fwd(m, ids[:0], ids[:0]).shape == (0, 200)
        p, keep = _struct_for(L, m)
        need = int(L.lib().kge_acre_trunk_workspace_bytes(ctypes.byref(p), ctypes.c_int64(2)))
        assert need > 0
        ws = torch.empty(need - 4, dtype=torch.uint8, device="cuda")
        x = torch.full((2, 200), 7.0, device="cuda")
        rc = L.lib().kge_acre_trunk_fwd(ctypes.byref(p), L._ptr(ids), L._ptr(ids), ctypes.c_int64(2), L._ptr(x),
                                        L._ptr(ws), ctypes.c_int64(ws.numel()), L._stream())
        assert rc == -4 and (x == 7.0).all()
        rc = L.lib().kge_acre_trunk_fwd(ctypes.byref(p), None, None, ctypes.c_int64(0), None, L._ptr(ws),
                                        ctypes.c_int64(ws.numel()), L._stream())
        assert rc == 0
        ws = torch.empty(need, dtype=torch.uint8, device="cuda")
        rc = L.lib().kge_acre_trunk_fwd(ctypes.byref(p), L._ptr(ids), L._ptr(ids), ctypes.c_int64(2), L._ptr(x),
                                        L._ptr(ws), ctypes.c_int64(ws.numel()), L._stream())
        assert rc == 0
    torch.cuda.synchronize()


# ---- the mirror vs the reference's outputs --------------------------------------------------------
@pytest.mark.parametrize("name", au.CASES)
def test_eval_forward_matches_reference(name):
    """model.forward(e, r, direction) in eval mode vs the reference's output: <= 1e-4 relative, x <= 1e-5"""
    g = au.load(name)
    m = au.mirror(g)
    h, r, t = _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])
    with torch.no_grad():
        pt = m(h, r, direction="tail").cpu().numpy()
        ph = m(t, r, direction="head").cpu().numpy()
        xt = m.proj_query(h, r, "tail").cpu().numpy()
        xh = m.proj_query(t, r, "head").cpu().numpy()
    assert gu.rel_err(pt, g["preds_tail"]).max() <= 1e-4 and gu.rel_err(ph, g["preds_head"]).max() <= 1e-4
    assert np.abs(xt - g["x_tail"]).max() <= 1e-5 and np.abs(xh - g["x_head"]).max() <= 1e-5
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


@pytest.mark.parametrize("name", au.CASES)
def test_evaluator_ranks_match_reference(name):
    g = au.load(name)
    m = au.mirror(g)
    Q = g["ranks"].shape[0]
    ev = _evaluator(m, int(g["N"]))
    with torch.no_grad():
        got = ev.rank_triples(g["h"][:Q], g["r"][:Q], g["t"][:Q], (g["filt_t_ptr"], g["filt_t_idx"]),
                              (g["filt_h_ptr"], g["filt_h_idx"]))
        assert ev.last_d2h_bytes == 16 * Q
        raw = ev.rank_triples(g["h"][:Q], g["r"][:Q], g["t"][:Q])
    assert np.array_equal(got, g["ranks"])
    assert np.array_equal(raw[:, 0], g["ranks"][:, 0]) and np.array_equal(raw[:, 2], g["ranks"][:, 2])
    assert np.array_equal(raw[:, 1], raw[:, 0]) and np.array_equal(raw[:, 3], raw[:, 2])


@pytest.mark.parametrize("cfg", au.FB237_CONFIGS, ids=_cfg_id)
def test_fb15k237_ranks_equal_the_oracle(fb237_models, cfg):
    """Evaluator.rank_triples at N = 14,541 (64 queries, filtered) == the oracle's trunk + oracle rank counts"""
    st, m = fb237_models[cfg]
    Q, N = 64, FB237["N"]
    rng = np.random.RandomState(11)
    h, r, t = rng.randint(N, size=Q), rng.randint(FB237["R"], size=Q), rng.randint(N, size=Q)
    ft = [np.unique(np.append(rng.randint(N, size=5), t[q])) for q in range(Q)]
    fh = [np.unique(np.append(rng.randint(N, size=5), h[q])) for q in range(Q)]
    csr = lambda rows: (np.concatenate([[0], np.cumsum([len(x) for x in rows])]).astype(np.int64),
                        np.concatenate(rows).astype(np.int64))
    ftc, fhc = csr(ft), csr(fh)
    with torch.no_grad():
        got = _evaluator(m, N).rank_triples(h, r, t, ftc, fhc)
    E, b = st["ent_embeddings.weight"], st["bias"]
    want = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(au.oracle_trunk_fwd(st, h, r), E, b, t, ftc, 0, want)
    oracle.proj_rank(au.oracle_trunk_fwd(st, t, r), E, b, h, fhc, 1, want)
    assert np.array_equal(got, want)


@pytest.mark.parametrize("name", au.CASES)
def test_training_step_matches_reference_autograd(name):
    """train_step_projection (trainer.py:159-174): loss and the gradient of every parameter vs the reference's
    own backward (fc.weight / W_gate_e.weight on the stored sample of entries and the row sums); BatchNorm
    running statistics after the two forwards."""
    from pykg2vec_b200.trainer import Trainer
    g = au.load(name)
    m = au.mirror(g, train=True)
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
        got = p.grad.detach().cpu().numpy()
        if "grad_" + key in g:
            want = g["grad_" + key]
            # conv / bn0 / fc biases in front of a training-mode BatchNorm have a true gradient of 0: relative
            # bound + floor
            assert np.abs(got - want).max() <= 5e-4 * np.abs(want).max() + 1e-7, key
        else:
            want = g["grad_sample_" + key]
            assert np.abs(got.reshape(-1)[g["grad_idx_" + key]] - want).max() <= 5e-4 * np.abs(want).max() + 1e-7, key
            rs, wrs = got.astype(np.float64).sum(1), g["grad_rowsum_" + key]
            assert np.abs(rs - wrs).max() <= 5e-4 * np.abs(wrs).max() + 1e-6, key
        seen.add(key)
    assert seen == {k[5:] for k in g if k.startswith("grad_") and not k.startswith(("grad_idx_", "grad_sample_",
                                                                                     "grad_rowsum_"))} | \
        {k[len("grad_idx_"):] for k in g if k.startswith("grad_idx_")}
    assert m.conv3.weight.grad.abs().max() > 0
    for key, v in m.state_dict().items():
        if "running" in key:
            assert np.abs(v.cpu().numpy() - g["sd_after_" + key]).max() < 1e-5, key


@pytest.mark.parametrize("way", ["serial", "parallel"])
def test_epoch_on_device_generator(way):
    """Generator (device label rows) -> Trainer.train_model_epoch -> batched Evaluator, AcrE, adam"""
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.generator import Generator
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    from pykg2vec_b200.trainer import Trainer
    kg = SyntheticKnowledgeGraph(200, 5, 2000, 60, 60, seed=3)
    cfg = SyntheticConfig(kg, device="cuda", optimizer="adam", learning_rate=0.003, batch_size=64, neg_rate=0,
                          hidden_size=200, in_channels=8, way=way, first_atrous=1, second_atrous=2,
                          third_atrous=2, acre_bias=True, input_dropout=0.0, feature_map_dropout=0.0,
                          hidden_dropout=0.0, label_smoothing=0.1, test_num=50)
    torch.manual_seed(0)
    model = import_model("acre")(**cfg.__dict__)
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
# hidden_size 200: the reference's trunk views each row as 10 x 20 (the CLI default of 50 cannot run)
argv = ["-mn", "acre", "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1", "-ds", "syn", "-dsp", ds,
        "-device", "cuda", "-k", "200", "-ic", "4"]
tr = du.run_cli_flow(argv, B200Importer)
out = {"cls": type(tr.model).__module__ + "." + type(tr.model).__name__, "cuda": next(tr.model.parameters()).is_cuda,
       "cfg": [tr.model.way, tr.model.in_channels, tr.model.hidden_size],
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
def test_reference_trainer_drives_acre(tmp_path):
    """the unmodified reference CLI flow (Importer -> Trainer.build_model / train_model -> Evaluator -> infer_*)
    with this package's AcrE patched into Importer, -device cuda"""
    import json
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    env = dict(os.environ, PYTHONPATH=os.pathsep.join([os.path.dirname(here), here, os.environ.get("PYTHONPATH", "")]))
    res = subprocess.run([sys.executable, "-c", DROPIN_FLOW], cwd=str(tmp_path), env=env, capture_output=True,
                         text=True, timeout=600)
    lines = [l for l in res.stdout.splitlines() if l.startswith("RESULT ")]
    assert res.returncode == 0 and lines, res.stderr[-4000:]
    out = json.loads(lines[-1][len("RESULT "):])
    assert out["cls"] == "pykg2vec_b200.projection.AcrE" and out["cuda"]
    assert len(out["losses"]) == 2 and np.isfinite(out["losses"]).all()
    assert out["losses"][1] < out["losses"][0]          # the loss goes down between the two epochs
    assert out["mr_finite"] and out["infer"] == [5, 5]
    assert out["rank_mismatch"] < 0.02, out["rank_mismatch"]   # only exact ties may order differently under topk
