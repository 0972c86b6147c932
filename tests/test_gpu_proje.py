"""GPU tests of ProjE_pointwise: the trunk kernel bit for bit against the oracle, the fused training step against
the oracle (fp32 and fp64), the reference's autograd and the autograd forward() path, Adam through both Trainer
paths, the Evaluator's ranks, dropout, the device Generator's negative labels, the unmodified reference Trainer
driving the class, and the C-ABI's argument errors."""
import ctypes
import types

import numpy as np
import pytest
import torch

import dropin_util as du
import oracle
import proje_util as pu

pytestmark = pytest.mark.gpu


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _bits_equal(a, b):
    return np.array_equal(np.asarray(a, np.float32).view(np.uint32), np.asarray(b, np.float32).view(np.uint32))


def _tabs_cuda(tabs):
    return [_cuda(t) for t in tabs]


def _fb15k237_tables(seed, N=14541, R=237, k=200):
    rng = np.random.RandomState(seed)
    xav = lambda rows, cols: (rng.uniform(-1, 1, (rows, cols)) * np.sqrt(6.0 / (rows + cols))).astype(np.float32)
    return [xav(N, k), xav(R, k)] + [xav(1, k) for _ in range(6)]


@pytest.mark.parametrize("name", pu.CASES)
def test_trunk_kernel_bit_exact_vs_oracle_on_goldens(name):
    from pykg2vec_b200 import _lib
    g = pu.load(name)
    tabs = pu.tables(pu.state(g))
    dt = _tabs_cuda(tabs)
    for d, (tag, e) in enumerate((("tail", g["h"]), ("head", g["t"]))):
        x = _lib.proje_trunk_fwd(dt, _cuda(e), _cuda(g["r"]), d).cpu().numpy()
        assert _bits_equal(x, pu.oracle_trunk(tabs, e, g["r"], d))
        assert np.abs(x - g["x_" + tag]).max() <= 1e-6
        nz = g["noise_" + tag]
        x = _lib.proje_trunk_fwd(dt, _cuda(e), _cuda(g["r"]), d, noise=_cuda(nz)).cpu().numpy()
        assert _bits_equal(x, pu.oracle_trunk(tabs, e, g["r"], d, nz))


@pytest.mark.parametrize("Q", [1, 77, 512])
def test_trunk_kernel_bit_exact_at_fb15k237_shape(Q):
    from pykg2vec_b200 import _lib
    tabs = _fb15k237_tables(Q)
    rng = np.random.RandomState(Q + 1)
    e, r = rng.randint(14541, size=Q), rng.randint(237, size=Q)
    dt = _tabs_cuda(tabs)
    for d in (0, 1):
        x = _lib.proje_trunk_fwd(dt, _cuda(e.astype(np.int64)), _cuda(r.astype(np.int64)), d).cpu().numpy()
        assert _bits_equal(x, pu.oracle_trunk(tabs, e, r, d))


def _fused_grads(dt, g, lt="lab_tail", lh="lab_head"):
    from pykg2vec_b200 import _lib
    grads = [torch.zeros_like(t) for t in dt]
    nt, nh = pu.noise_or_none(g, "tail"), pu.noise_or_none(g, "head")
    loss = _lib.proje_train_step(dt, _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"]), _cuda(g[lt]), _cuda(g[lh]), grads,
                                 _cuda(nt) if nt is not None else None, _cuda(nh) if nh is not None else None)
    reg = _lib.reg_l1_dense([dt[i] for i in pu.REG_INDEX], [grads[i] for i in pu.REG_INDEX], float(g["lmbda"]))
    return float(loss.item()), float(reg.item()), [x.cpu().numpy() for x in grads]


@pytest.mark.parametrize("name", pu.CASES)
def test_fused_step_matches_oracle_and_reference(name):
    g = pu.load(name)
    tabs = pu.tables(pu.state(g))
    loss, reg, grads = _fused_grads(_tabs_cuda(tabs), g)
    nt, nh = pu.noise_or_none(g, "tail"), pu.noise_or_none(g, "head")
    wloss, _ = pu.oracle_step(tabs, g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"], nt, nh)
    assert abs(loss - wloss) <= 1e-5 * abs(wloss)
    want = float(g["loss_tail"]) + float(g["loss_head"])
    assert abs(loss - want) <= 1e-5 * abs(want)
    assert abs(reg - float(g["reg"])) <= 1e-5 * abs(float(g["reg"]))
    for key, a, b in zip(pu.KEYS, grads, pu.golden_grads(g)):
        assert np.abs(a - b).max() <= 5e-4 * np.abs(b).max() + 1e-7, key
    if name != "proje_heavy":     # fp64 does not saturate where fp32 does
        _, w64 = pu.oracle_step(tabs, g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"], nt, nh, fp64=True)
        pu.oracle_reg(tabs, float(g["lmbda"]), w64)
        for key, a, b in zip(pu.KEYS, grads, w64):
            assert np.abs(a - b).max() <= 1e-4 * np.abs(b).max() + 1e-7, key


@pytest.mark.parametrize("name", pu.CASES)
def test_autograd_forward_matches_fused_step(name):
    """forward(e, r, er_e2, direction) + get_reg through loss.backward() == the fused step + regulariser, with the
    recorded noise in both (the mirror's dropout draw replaced by the golden's)"""
    g = pu.load(name)
    m = pu.mirror(g)
    noises = iter([pu.noise_or_none(g, "tail"), pu.noise_or_none(g, "head")])
    m.dropout_noise = lambda rows: (lambda n: _cuda(n) if n is not None else None)(next(noises))
    m.zero_grad()
    lt = m(_cuda(g["h"]), _cuda(g["r"]), _cuda(g["lab_tail"]), direction="tail")
    lh = m(_cuda(g["t"]), _cuda(g["r"]), _cuda(g["lab_head"]), direction="head")
    loss = m.loss(lh, lt) + m.get_reg(None, None, None)
    loss.backward()
    floss, freg, fgrads = _fused_grads(_tabs_cuda(pu.tables(pu.state(g))), g)
    assert abs(loss.item() - (floss + freg)) <= 1e-5 * abs(floss + freg)
    for key, a, b in zip(pu.KEYS, [p.weight.grad.cpu().numpy() for p in m.parameter_list], fgrads):
        assert np.abs(a - b).max() <= 1e-5 * np.abs(b).max() + 1e-7, key


def _trainer(g, fused, seed):
    from pykg2vec_b200.trainer import Trainer
    torch.manual_seed(seed)
    m = pu.mirror(g)
    cfg = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=0.01, fused_step=fused,
                                tot_entity=int(g["N"]), batch_size=len(g["h"]), knowledge_graph=None)
    tr = Trainer(m, cfg)
    import pykg2vec_b200.trainer as trmod
    ev = trmod.Evaluator
    trmod.Evaluator = lambda *a, **k: None     # no evaluation here: the config carries no knowledge graph
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev
    return tr


@pytest.mark.parametrize("name", ["proje_n60", "proje_n300"])
def test_three_adam_steps_fused_and_autograd_agree(name):
    g = pu.load(name)
    a, b = _trainer(g, True, 0), _trainer(g, False, 0)
    assert a._proje and not b._proje
    batch = [g["h"], g["r"], g["t"], g["lab_tail"], g["lab_head"]]
    for step in range(3):
        torch.manual_seed(100 + step)     # the same dropout draws on both paths
        la = a.train_batch(batch)
        torch.manual_seed(100 + step)
        lb = b.train_batch(batch)
        assert abs(la - lb) <= 1e-5 * abs(lb)
    for key, pa, pb in zip(pu.KEYS, a.model.parameter_list, b.model.parameter_list):
        d = np.abs(pa.weight.detach().cpu().numpy() - pb.weight.detach().cpu().numpy())
        # an element whose gradient cancels to rounding noise may take a different Adam step: bound the rest
        assert d.max() <= 6 * 0.01 and (d <= 1e-5).mean() >= 0.999, key


@pytest.mark.parametrize("name", pu.CASES)
def test_evaluator_ranks_match_reference_and_oracle(name):
    from pykg2vec_b200.evaluator import Evaluator
    g = pu.load(name)
    m = pu.mirror(g).eval()
    Q = g["ranks"].shape[0]
    h, r, t = g["h"][:Q], g["r"][:Q], g["t"][:Q]
    ev = object.__new__(Evaluator)
    ev.model, ev.config = m, types.SimpleNamespace(device="cuda", tot_entity=int(g["N"]))
    ev._filter_cache, ev._workspace = {}, None
    ft, fh = (g["filt_t_ptr"], g["filt_t_idx"]), (g["filt_h_ptr"], g["filt_h_idx"])
    with torch.no_grad():
        got = ev.rank_triples(h, r, t, ft, fh)
    assert np.array_equal(got, g["ranks"])
    tabs = pu.tables(pu.state(g))
    want = np.zeros((Q, 4), dtype=np.int32)
    oracle.proj_rank(pu.oracle_trunk(tabs, h, r, 0), tabs[0], None, t, ft, 0, want)
    oracle.proj_rank(pu.oracle_trunk(tabs, t, r, 1), tabs[0], None, h, fh, 1, want)
    assert np.array_equal(got, want)
    # predict_*_rank of the mirror: the target's position in topk(-preds) is at least the count of better entities
    rank = m.predict_tail_rank(_cuda(h[:1]), _cuda(r[:1]), topk=int(g["N"])).cpu().numpy()
    assert rank.shape == (1, int(g["N"])) and sorted(rank[0].tolist()) == list(range(int(g["N"])))


def test_dropout_noise_fraction_and_scale():
    from pykg2vec_b200 import import_model
    m = import_model("proje_pointwise")(tot_entity=50, tot_relation=3, hidden_size=200, lmbda=1e-5, hidden_dropout=0.3,
                                        device="cuda").cuda()
    n = m.dropout_noise(4000).cpu().numpy()
    vals = set(np.unique(n).tolist())
    assert vals == {0.0, float(np.float32(1.0) / np.float32(0.7))}
    kept, total = (n != 0).sum(), n.size
    sd = np.sqrt(total * 0.7 * 0.3)
    assert abs(kept - 0.7 * total) <= 6 * sd
    m.hidden_dropout = 0.0
    assert m.dropout_noise(10) is None


def _synthetic(neg_rate, dropout=0.5):
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(300, 5, 3000, 60, 60, seed=3)
    return SyntheticConfig(kg, device="cuda", optimizer="adam", learning_rate=0.01, batch_size=64, neg_rate=neg_rate,
                           hidden_size=32, hidden_dropout=dropout, lmbda=1e-5, test_num=50)


def test_generator_negative_labels_rule():
    """every row of both directions: -1 at the same 100 distinct ids unless they are its positives, the positives
    exactly those of the positives-only label rows"""
    from pykg2vec_b200 import _lib, import_model
    from pykg2vec_b200.generator import Generator
    cfg = _synthetic(1)
    model = import_model("proje_pointwise")(**cfg.__dict__)
    gen = Generator(model, cfg, seed=2)
    gen.start_one_epoch(1)
    sel = gen._perm[:64]
    h, r, t, hr_t, tr_h = next(gen)
    cand = None
    for lab, csr in ((hr_t, gen._hr), (tr_h, gen._tr)):
        lab = lab.cpu().numpy()
        pos = _lib.proj_labels(csr[0][sel], csr[1], csr[2], 64, 300).cpu().numpy()
        assert np.array_equal(lab == 1, pos == 1)                   # positives never overwritten
        assert set(np.unique(lab).tolist()) <= {-1.0, 0.0, 1.0}
        neg = set(np.nonzero((lab == -1).any(axis=0))[0].tolist())
        cand = neg if cand is None else cand | neg
        for b in range(64):
            assert set(np.nonzero(lab[b] == -1)[0].tolist()) <= neg
    cols = np.array(sorted(cand))
    assert len(cols) == 100                                         # min(100, N) shared ids, N = 300
    for lab in (hr_t.cpu().numpy(), tr_h.cpu().numpy()):
        assert (lab[:, cols] != 0).all()                            # each is -1 or a positive in every row


def test_epoch_on_device_generator():
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.generator import Generator
    from pykg2vec_b200.trainer import Trainer
    cfg = _synthetic(1)
    torch.manual_seed(0)
    model = import_model("proje_pointwise")(**cfg.__dict__)
    tr = Trainer(model, cfg)
    tr.build_model()
    assert tr._proje
    gen = Generator(model, cfg, seed=1)
    losses = [tr.train_model_epoch(gen, num_batch=10) for _ in range(4)]
    assert all(np.isfinite(losses)) and losses[-1] < losses[0]
    model.eval()
    scores = tr.evaluator.mini_test(epoch=0)
    assert set(scores) == {"mr", "fmr", "mrr", "fmrr"} and 1.0 <= scores["fmr"] <= scores["mr"] <= 300.0


def test_argument_errors_and_empty_batches():
    from pykg2vec_b200 import _lib
    L = _lib.lib()
    tabs = _tabs_cuda(_fb15k237_tables(0, N=50, R=4, k=8))
    p = _lib.proje_struct(tabs)
    ids = torch.zeros(4, dtype=torch.int64, device="cuda")
    x = torch.empty((4, 8), device="cuda")
    s = _lib._stream()
    P = ctypes.byref(p)
    assert L.kge_proje_trunk_fwd(P, 2, _lib._ptr(ids), _lib._ptr(ids), ctypes.c_int64(4), None, _lib._ptr(x), s) == -1
    assert L.kge_proje_trunk_fwd(None, 0, _lib._ptr(ids), _lib._ptr(ids), ctypes.c_int64(4), None, _lib._ptr(x), s) == -1
    assert L.kge_proje_trunk_fwd(P, 0, _lib._ptr(ids), _lib._ptr(ids), ctypes.c_int64(-1), None, _lib._ptr(x), s) == -1
    assert L.kge_proje_trunk_fwd(P, 0, None, None, ctypes.c_int64(0), None, None, s) == 0     # Q = 0: no-op
    wide = _lib.proje_struct(_tabs_cuda(_fb15k237_tables(0, N=4, R=2, k=1028)))
    assert L.kge_proje_trunk_fwd(ctypes.byref(wide), 0, _lib._ptr(ids), _lib._ptr(ids), ctypes.c_int64(1), None,
                                 _lib._ptr(x), s) == -2
    loss = torch.full((1,), 7.0, device="cuda")
    grads = _lib._table_ptr_array([None] * 8)
    lab = torch.zeros((4, 50), device="cuda")
    step = lambda *a: L.kge_proje_train_step(*a, grads, _lib._ptr(loss), s)
    assert step(P, _lib._ptr(ids), _lib._ptr(ids), _lib._ptr(ids), ctypes.c_int64(4), None, None, None, None) == -1
    assert step(P, None, _lib._ptr(ids), None, ctypes.c_int64(4), _lib._ptr(lab), None, None, None) == -1
    assert step(P, None, None, None, ctypes.c_int64(0), _lib._ptr(lab), None, None, None) == 0
    assert loss.item() == 0.0                                  # an empty batch has a zero loss
    assert L.kge_reg_l1_dense(None, None, None, 1, ctypes.c_float(1.0), _lib._ptr(loss), s) == -1
    assert L.kge_proj_labels_negatives(_lib._ptr(lab), ctypes.c_int64(4), ctypes.c_int64(50), _lib._ptr(ids),
                                       ctypes.c_int64(51), s) == -1
    assert L.kge_proj_labels_negatives(None, ctypes.c_int64(0), ctypes.c_int64(50), None, ctypes.c_int64(5), s) == 0
    torch.cuda.synchronize()


# The reference's Generator forks its worker processes; a fork taken after this test process has run OpenMP
# regions (the oracle) can deadlock the child, so the reference's flow runs in a fresh interpreter.
DROPIN_FLOW = r"""
import json, os, sys
import numpy as np
import torch
import dropin_util as du
B200Importer = du.b200_importer_class()
ds = du.write_dataset(os.path.abspath("data"))
argv = ["-mn", "proje_pointwise", "-l", "2", "-ts", "1", "-tn", "50", "-npg", "1", "-ds", "syn", "-dsp", ds,
        "-device", "cuda", "-k", "32", "-lmda", "1e-5", "-hdt", "0.5", "-ngr", "1"]
tr = du.run_cli_flow(argv, B200Importer)
out = {"cls": type(tr.model).__module__ + "." + type(tr.model).__name__, "cuda": next(tr.model.parameters()).is_cuda,
       "losses": [float(v) for _, v in tr.training_results],
       "mr_finite": all(bool(np.isfinite(v)) for v in tr.evaluator.metric_calculator.mr.values()),
       "infer": [len(tr.infer_tails(1, 10, topk=5)), len(tr.infer_heads(10, 20, topk=5))]}
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
def test_reference_trainer_drives_proje(tmp_path):
    """the unmodified reference CLI flow (Importer -> Trainer.build_model / train_model -> Evaluator -> infer_*)
    with this package's ProjE_pointwise patched into Importer, -device cuda, neg_rate 1"""
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
    assert out["cls"] == "pykg2vec_b200.projection.ProjE_pointwise" and out["cuda"]
    assert len(out["losses"]) == 2 and np.isfinite(out["losses"]).all()
    assert out["mr_finite"] and out["infer"] == [5, 5]
    assert out["rank_mismatch"] < 0.02, out["rank_mismatch"]   # only exact ties may order differently under topk
