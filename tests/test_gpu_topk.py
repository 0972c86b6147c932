"""H100 tests of batched top-k link prediction (kge_topk_1vsall, kge_proj_topk, Evaluator.predict_*): exact ids and
bit-exact scores against the oracle's scores plus the numpy selection of tests/topk_util.py, for every kernel model
(tails, heads, relations; raw and filtered; k = 1, 10, 256), dataset-sized tables, query counts that cross the
Evaluator's batches and the launchers' internal chunks, the six projection models, and a cross-check of the target's
position against the independent rank-counting kernels."""
import types

import numpy as np
import pytest
import torch

import golden_util as gu
import gpu_util as gpu
import oracle
from topk_util import csr, ref_topk

pytestmark = pytest.mark.gpu

KS = (1, 10, 256)


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.int64)).cuda()


def _oracle_scores(om, target, h, r, t):
    if target == 0:
        return oracle.sweep_scores(om, oracle.GROUP_TAIL, h, r, t)
    if target == 1:
        return oracle.sweep_scores(om, oracle.GROUP_HEAD, h, r, t)
    n = om.num_rel
    return oracle.score_fwd(om, np.full(n, h), np.arange(n), np.full(n, t), oracle.GROUP_TAIL)


def _check(om, desc, target, qh, qr, qt, k, filt_rows=None):
    from pykg2vec_b200 import _lib
    f = None
    if filt_rows is not None:
        p, i = csr(filt_rows)
        f = (_cuda(p), _cuda(i))
    ids, sc = _lib.topk_1vsall(desc, target, _cuda(qh), _cuda(qr), _cuda(qt), k, f)
    ids, bits = ids.cpu().numpy(), sc.cpu().numpy().view(np.uint32)
    for q in range(len(qh)):
        s = _oracle_scores(om, target, qh[q], qr[q], qt[q])
        want_ids, want_bits = ref_topk(s, k, filt=filt_rows[q] if filt_rows is not None else None)
        assert np.array_equal(ids[q], want_ids), (target, k, q, ids[q][:8], want_ids[:8])
        assert np.array_equal(bits[q], want_bits), (target, k, q)


@pytest.mark.parametrize("name", gu.case_names())
def test_every_kernel_model_at_its_golden_tables(name):
    g = gu.load(name)
    om = gu.oracle_model(g)
    if om.name == "rescal":            # what Rescal.forward (and the Evaluator) does to the tables first
        for tab in om.tables:
            oracle.normalize_rows(tab)
    desc = gpu.desc_from_oracle_model(om)
    Q = 6
    qh, qr, qt = (np.ascontiguousarray(g[k][:Q], dtype=np.int64) for k in ("h", "r", "t"))
    rng = np.random.RandomState(0)
    for target in (0, 1, 2):
        n = om.num_rel if target == 2 else om.num_ent
        filt = [rng.randint(n, size=rng.randint(0, n)).tolist() + [0, 0] for _ in range(Q)]   # duplicates included
        for k in KS:
            _check(om, desc, target, qh, qr, qt, k)
            _check(om, desc, target, qh, qr, qt, k, filt)


@pytest.mark.parametrize("model,N,d", [("transe", 14541, 200), ("distmult", 14541, 200), ("complex", 14541, 200),
                                       ("rotate", 14541, 200), ("transe", 123182, 64)])
def test_dataset_sized_tables(model, N, d):
    om, _ = gpu.synthetic_case(model, N, 237, d, seed=11, margin=6.0 if model == "rotate" else 0.0, scale=0.3)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(1)
    Q = 5
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(237, size=Q), rng.randint(N, size=Q)
    filt = [rng.randint(N, size=400).tolist() for _ in range(Q)]
    for target in (0, 1):
        for k in (10, 256):
            _check(om, desc, target, qh, qr, qt, k, filt if k == 256 else None)
    _check(om, desc, 2, qh, qr, qt, 10)


def test_query_counts_cross_batches_and_chunks():
    """Q = 1, 513 and 70,000: the Evaluator's QUERY_BATCH and the launcher's 64 MiB chunks (8,388 rows at N = 2,000)"""
    from pykg2vec_b200 import _lib
    from pykg2vec_b200.evaluator import Evaluator
    N, R, d, k = 2000, 11, 16, 10
    om, _ = gpu.synthetic_case("transe", N, R, d, seed=5)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(2)
    ev = Evaluator.__new__(Evaluator)
    ev.QUERY_BATCH = 8192
    ev.model = types.SimpleNamespace(kge_desc=lambda: desc)
    ev.config = types.SimpleNamespace(device="cuda", tot_entity=N, tot_relation=R)
    for Q in (1, 513, 70000):
        qh, qr = rng.randint(N, size=Q), rng.randint(R, size=Q)
        S = np.stack([oracle.sweep_scores(om, oracle.GROUP_TAIL, qh[q], qr[q], 0) for q in range(Q)])
        want = np.argsort(S, axis=1, kind="stable")[:, :k]     # TransE distances: no NaN, no -0
        ids, sc = ev.predict_tails(qh, qr, k=k)
        assert ids.shape == (Q, k) and sc.dtype == np.float32
        assert np.array_equal(ids, want), Q
        assert np.array_equal(sc.view(np.uint32), np.take_along_axis(S, want, 1).view(np.uint32))
        if Q == 70000:   # one kernel call over every query: nine internal chunks
            i2, s2 = _lib.topk_1vsall(desc, 0, _cuda(qh), _cuda(qr), None, k)
            assert np.array_equal(i2.cpu().numpy(), want)


def test_constant_tables_give_the_smallest_ids():
    from pykg2vec_b200 import _lib
    om, tabs = gpu.synthetic_case("distmult", 3000, 5, 32, seed=0)
    for t in om.tables:
        t[...] = 0.5
    desc = gpu.desc_from_oracle_model(om)
    q = _cuda(np.array([0, 7, 2999]))
    for target in (0, 1, 2):
        for k in KS:
            ids, sc = _lib.topk_1vsall(desc, target, q, _cuda(np.array([0, 1, 4])), q, k)
            n = 5 if target == 2 else 3000
            want = np.tile(np.r_[np.arange(min(k, n)), -np.ones(max(0, k - n), np.int64)], (3, 1))
            assert np.array_equal(ids.cpu().numpy(), want), (target, k)


def _trained_kg_model(name, N=300, R=7):
    import pykg2vec_b200
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(N, R, 1500, 50, 50, seed=4)
    cfg = SyntheticConfig(kg, hidden_size=24, l1_flag=False, num_filters=4, filter_sizes=[1, 2, 3])
    torch.manual_seed(0)
    m = pykg2vec_b200.import_model(name)(**cfg.__dict__).cuda()
    return kg, cfg, m


@pytest.mark.parametrize("name", ["transe", "complex", "rescal", "convkb"])
def test_position_of_the_target_equals_its_rank(name):
    """On tie-free queries the target's place in predict_* output is rank_triples' count: two independent kernels.
    Rescal's in-place normalisation and ConvKB's derived tables go through the same per-call preparation."""
    from pykg2vec_b200.evaluator import Evaluator
    kg, cfg, m = _trained_kg_model(name)
    ev = Evaluator(m, cfg)
    arr = kg.arrays["test"][:40]
    hs, rs, ts = arr[:, 0], arr[:, 1], arr[:, 2]
    ranks = ev.rank_triples(hs, rs, ts)
    k = 256
    ti, tsc = ev.predict_tails(hs, rs, k=k)
    hi, hsc = ev.predict_heads(rs, ts, k=k)
    fti, _ = ev.predict_tails(hs, rs, k=k, filtered=True)
    checked = 0
    for q in range(len(hs)):
        for ids, sc, tgt, col in ((ti, tsc, ts, 0), (hi, hsc, hs, 2)):
            if len(np.unique(sc[q].view(np.uint32))) != k or tgt[q] not in ids[q]:
                continue   # ties or the target beyond k: positions are not ranks
            assert list(ids[q]).index(tgt[q]) == ranks[q, col], (name, q, col)
            checked += 1
        assert not set(fti[q].tolist()) & ev.metric_calculator.hr_t[(int(hs[q]), int(rs[q]))]
    assert checked >= 10


def test_filtered_position_equals_filtered_rank():
    """The filtered list (target re-admitted by removing it from the CSR) places the target at rank_triples' filtered
    count."""
    from pykg2vec_b200 import _lib
    from pykg2vec_b200.evaluator import Evaluator, build_filter_csr
    kg, cfg, m = _trained_kg_model("distmult")
    ev = Evaluator(m, cfg)
    arr = kg.arrays["test"][:40]
    hs, rs, ts = arr[:, 0], arr[:, 1], arr[:, 2]
    keys = [(int(h), int(r)) for h, r in zip(hs, rs)]
    ft = build_filter_csr(keys, {key: ev.metric_calculator.hr_t[key] - {int(t)} for key, t in zip(keys, ts)})
    fh = build_filter_csr([(int(t), int(r)) for t, r in zip(ts, rs)], {})
    counts = ev.rank_triples(hs, rs, ts, ft, fh)
    ids, sc = _lib.topk_1vsall(m.kge_desc(), 0, _cuda(hs), _cuda(rs), None, 256, (_cuda(ft[0]), _cuda(ft[1])))
    ids, sc = ids.cpu().numpy(), sc.cpu().numpy()
    checked = 0
    for q in range(len(hs)):
        valid = ids[q] >= 0
        if len(np.unique(sc[q][valid].view(np.uint32))) != valid.sum() or ts[q] not in ids[q]:
            continue
        assert list(ids[q]).index(ts[q]) == counts[q, 1]
        checked += 1
    assert checked >= 10


PROJ_CONFIGS = {
    "conve": dict(hidden_size=50, hidden_size_1=5),
    "tucker": dict(ent_hidden_size=32, rel_hidden_size=16, hidden_dropout1=0.0, hidden_dropout2=0.0),
    "hyper": dict(ent_hidden_size=32, rel_hidden_size=16),
    "interacte": dict(hidden_size=24, feature_permutation=2, num_filters=8, kernel_size=5, reshape_height=6,
                      reshape_width=4),
    "acre": dict(hidden_size=200, in_channels=8, way="serial", first_atrous=1, second_atrous=2, third_atrous=2,
                 acre_bias=True),
    "proje_pointwise": dict(hidden_size=32),
}


@pytest.mark.parametrize("name", sorted(PROJ_CONFIGS))
def test_projection_models_through_the_evaluator(name):
    import pykg2vec_b200
    from pykg2vec_b200 import _lib
    from pykg2vec_b200.evaluator import Evaluator
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    N, R = 400, 6
    kg = SyntheticKnowledgeGraph(N, R, 3000, 50, 50, seed=7)
    cfg = SyntheticConfig(kg, device="cuda", input_dropout=0.0, hidden_dropout=0.0, feature_map_dropout=0.0,
                          label_smoothing=0.1, lmbda=0.1, **PROJ_CONFIGS[name])
    torch.manual_seed(0)
    m = pykg2vec_b200.import_model(name)(**cfg.__dict__).cuda().eval()
    ev = Evaluator(m, cfg)
    arr = kg.arrays["test"][:30]
    hs, rs, ts = arr[:, 0], arr[:, 1], arr[:, 2]
    ent, bias = m.proj_tail_tables()
    ent = ent.detach().cpu().numpy()
    bias = bias.detach().cpu().numpy() if bias is not None else None
    make_cores = getattr(m, "proj_query_cores", None)
    with torch.no_grad():
        cores = make_cores(torch.from_numpy(np.unique(rs)).cuda()) if make_cores is not None else None
        kw = {"cores": cores} if cores is not None else {}
        x_t = m.proj_query(_cuda(hs), _cuda(rs), direction="tail", **kw).cpu().numpy()
        x_h = m.proj_query(_cuda(ts), _cuda(rs), direction="head", **kw).cpu().numpy()
    for k in (1, 10, 256):
        for filtered in (False, True):
            got = (ev.predict_tails(hs, rs, k=k, filtered=filtered), ev.predict_heads(rs, ts, k=k, filtered=filtered))
            for (ids, sc), x, keys, dct in ((got[0], x_t, zip(hs, rs), ev.metric_calculator.hr_t),
                                            (got[1], x_h, zip(ts, rs), ev.metric_calculator.tr_h)):
                P = oracle.proj_tail_fwd(x, ent, bias)
                for q, key in enumerate(keys):
                    f = sorted(dct.get((int(key[0]), int(key[1])), ())) if filtered else None
                    want_ids, want_bits = ref_topk(P[q], k, descending=True, filt=f)
                    assert np.array_equal(ids[q], want_ids), (name, k, filtered, q)
                    assert np.array_equal(sc[q].view(np.uint32), want_bits), (name, k, filtered, q)
    with pytest.raises(_lib.KgeNotSupported):
        ev.predict_rels(hs, ts)


def test_refusals_happen_before_any_launch():
    from pykg2vec_b200 import _lib
    from pykg2vec_b200.evaluator import Evaluator
    kg, cfg, m = _trained_kg_model("transe")
    ev = Evaluator(m, cfg)
    before = _lib.launch_count()
    for call in (lambda: ev.predict_tails([0, 300], [0, 0]), lambda: ev.predict_heads([7], [0]),
                 lambda: ev.predict_rels([-1], [0]), lambda: ev.predict_tails([0], [0], k=0),
                 lambda: ev.predict_tails([0], [0], k=257)):
        with pytest.raises(ValueError):
            call()
    assert _lib.launch_count() == before
    ids, sc = ev.predict_rels([0, 1], [2, 3], k=10)   # 7 relations: the last three slots are empty
    assert np.all(ids[:, 7:] == -1) and np.all(np.isnan(sc[:, 7:])) and np.all(ids[:, :7] >= 0)
