"""-m gpu parity tests: CUDA path (through the C-ABI) vs the CPU oracle, bit-exact on
scores and exact on rank counts; and vs the golden outputs of the reference itself
(scores within 1e-4 relative, ranks exact)."""
import numpy as np
import pytest
import torch

import golden_util as gu
import gpu_util as gpu

pytestmark = pytest.mark.gpu
CASES = gu.case_names()


def _lib():
    from pykg2vec_b200 import _lib
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.mark.parametrize("name", CASES)
def test_score_fwd_golden(name):
    import oracle
    L = _lib()
    g = gu.load(name)
    desc = gpu.desc_from_golden(g)
    om = gu.oracle_model(g)
    h, r, t = _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])
    for grouping in (L.GROUP_TAIL, L.GROUP_HEAD):
        s = L.score_fwd(desc, h, r, t, grouping).cpu().numpy()
        so = oracle.score_fwd(om, g["h"], g["r"], g["t"], grouping)
        np.testing.assert_array_equal(gpu.bits(s), gpu.bits(so), err_msg="%s grouping %d: kernel != oracle bitwise" % (name, grouping))
        ref = g["scores"]
        floor = 1e-2 * np.abs(ref).max()
        err = np.abs(s.astype(np.float64) - ref) / np.maximum(np.abs(ref), floor)
        assert err.max() < 1e-4, (name, err.max())


@pytest.mark.parametrize("name", CASES)
@pytest.mark.parametrize("flags", [0, 1])
def test_rank_golden(name, flags):
    L = _lib()
    g = gu.load(name)
    desc = gpu.desc_from_golden(g)
    Q = g["ranks"].shape[0]
    counts = L.rank_1vsall(desc, _cuda(g["h"][:Q]), _cuda(g["r"][:Q]), _cuda(g["t"][:Q]),
                           (_cuda(g["filt_t_ptr"]), _cuda(g["filt_t_idx"])),
                           (_cuda(g["filt_h_ptr"]), _cuda(g["filt_h_idx"])), flags=flags)
    np.testing.assert_array_equal(counts.cpu().numpy(), g["ranks"])


SYN = [
    # name, N, R, d, dr, l1, margin
    ("transe", 1500, 13, 200, None, False, 0.0),
    ("transe", 1500, 13, 50, None, True, 0.0),
    ("transe", 700, 5, 37, None, True, 0.0),
    ("transm", 900, 7, 64, None, False, 0.0),
    ("transh", 900, 7, 100, None, False, 0.0),
    ("transd", 900, 7, 50, None, True, 0.0),
    ("transr", 400, 5, 40, 24, False, 0.0),
    ("rotate", 800, 9, 1000, None, False, 24.0),
    ("rotate", 800, 9, 50, None, False, 6.0),
    ("distmult", 1500, 11, 200, None, False, 0.0),
    ("cp", 900, 11, 30, None, False, 0.0),
    ("complex", 1500, 11, 200, None, False, 0.0),
    ("complex", 1200, 11, 500, None, False, 0.0),
    ("hole", 500, 7, 150, None, False, 0.0),
    ("hole", 400, 7, 32, None, False, 0.0),
    ("rescal", 500, 5, 48, None, False, 0.0),
    ("rescal", 300, 5, 50, None, False, 0.0),
    ("slm", 400, 5, 64, 32, False, 0.0),
    ("slm", 300, 5, 50, 30, False, 0.0),
    ("ntn", 200, 4, 32, 16, False, 0.0),
    ("ntn", 150, 4, 20, 20, False, 0.0),
    ("sme", 300, 5, 48, None, False, 0.0),
    ("sme_bl", 300, 5, 50, None, False, 0.0),
    ("kg2e", 500, 5, 100, None, False, 0.0),
    ("kg2e", 300, 5, 50, None, False, 0.0),
    ("quate", 400, 5, 100, None, False, 0.0),
    ("quate", 300, 5, 30, None, False, 0.0),
    ("octonione", 300, 5, 48, None, False, 0.0),
    ("analogy", 700, 7, 200, None, False, 0.0),
    ("analogy", 500, 7, 36, None, False, 0.0),
    ("simple", 900, 7, 200, None, False, 0.0),
    ("simple_ignr", 700, 7, 50, None, False, 0.0),
    ("convkb", 900, 7, 100, None, False, 0.0),
    ("convkb", 500, 5, 50, None, False, 0.0),
]


@pytest.mark.parametrize("spec", SYN, ids=lambda s: "%s-N%d-d%d" % (s[0], s[1], s[3]))
def test_score_and_rank_synthetic_bitexact(spec):
    import oracle
    L = _lib()
    name, N, R, d, dr, l1, margin = spec
    om, _ = gpu.synthetic_case(name, N, R, d, seed=hash(spec) % 10007, dr=dr, l1=l1, margin=margin)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(5)
    for n in (1, 31, 257, 1000):
        h, r, t = rng.randint(N, size=n), rng.randint(R, size=n), rng.randint(N, size=n)
        for grouping in (0, 1):
            s = L.score_fwd(desc, _cuda(h), _cuda(r), _cuda(t), grouping).cpu().numpy()
            so = oracle.score_fwd(om, h, r, t, grouping)
            np.testing.assert_array_equal(gpu.bits(s), gpu.bits(so))
    Q = 5
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    for flags in (0, 1):
        got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), (_cuda(ft[0]), _cuda(ft[1])),
                            (_cuda(fh[0]), _cuda(fh[1])), flags=flags).cpu().numpy()
        np.testing.assert_array_equal(got, want)


def test_empty_and_argument_errors():
    L = _lib()
    g = gu.load("transe_l1_d50")
    desc = gpu.desc_from_golden(g)
    e = torch.empty(0, dtype=torch.int64, device="cuda")
    assert L.score_fwd(desc, e, e, e).numel() == 0
    with pytest.raises(L.KgeError):
        L.score_fwd(desc, _cuda(g["h"]), _cuda(g["r"][:5]), _cuda(g["t"]))
    with pytest.raises(L.KgeError):
        L.score_fwd(desc, _cuda(g["h"]).int(), _cuda(g["r"]), _cuda(g["t"]))


def test_rank_row_shards_add_up():
    """partial counts over disjoint row shards (separate shard tables + compact query table)
    add up to the replicated result — the row-sharded multi-GPU formulation on one GPU."""
    L = _lib()
    import oracle
    om, tabs = gpu.synthetic_case("complex", 1000, 7, 100, seed=3)
    rng = np.random.RandomState(9)
    Q = 7
    qh, qr, qt = rng.randint(1000, size=Q), rng.randint(7, size=Q), rng.randint(1000, size=Q)
    ft, fh = gpu.random_filters_csr(rng, 1000, qh, qr, qt)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    # compact query table: rows of all query heads and tails, queries re-indexed into it
    uniq = np.unique(np.concatenate([qh, qt]))
    remap = {int(e): i for i, e in enumerate(uniq)}
    qtabs = [torch.from_numpy(tabs[0][uniq]).cuda(), torch.from_numpy(tabs[1][uniq]).cuda(),
             torch.from_numpy(tabs[2]).cuda(), torch.from_numpy(tabs[3]).cuda()]
    qdesc = L.ModelDesc("complex", qtabs, 100)
    qh2 = np.asarray([remap[int(e)] for e in qh]); qt2 = np.asarray([remap[int(e)] for e in qt])
    counts = torch.zeros((Q, 4), dtype=torch.int32, device="cuda")
    for lo, hi in ((0, 300), (300, 301), (301, 1000)):
        stabs = [torch.from_numpy(np.ascontiguousarray(tabs[0][lo:hi])).cuda(),
                 torch.from_numpy(np.ascontiguousarray(tabs[1][lo:hi])).cuda(), qtabs[2], qtabs[3]]
        sdesc = L.ModelDesc("complex", stabs, 100)
        L.rank_1vsall(sdesc, _cuda(qh2), _cuda(qr), _cuda(qt2), (_cuda(ft[0]), _cuda(ft[1])),
                      (_cuda(fh[0]), _cuda(fh[1])), counts=counts, row_lo=lo, row_hi=hi, query_desc=qdesc,
                      tgt_h=_cuda(qh), tgt_t=_cuda(qt))
    np.testing.assert_array_equal(counts.cpu().numpy(), want)


@pytest.mark.parametrize("name,N,R,d", [("transe", 1, 1, 4), ("transe", 5, 2, 3), ("distmult", 33, 1, 1),
                                        ("complex", 31, 3, 2), ("rotate", 65, 2, 6), ("transh", 2, 1, 5)])
def test_tiny_and_ragged_shapes(name, N, R, d):
    """degenerate geometries: fewer entities than one candidate tile, widths below one 16-byte
    chunk, a single entity (every rank is 0), Q not a multiple of the query block."""
    import oracle
    L = _lib()
    om, _ = gpu.synthetic_case(name, N, R, d, seed=N * 7 + d, margin=3.0 if name == "rotate" else 0.0)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(d)
    Q = 67
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    s = L.score_fwd(desc, _cuda(qh), _cuda(qr), _cuda(qt)).cpu().numpy()
    np.testing.assert_array_equal(gpu.bits(s), gpu.bits(oracle.score_fwd(om, qh, qr, qt)))
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=3)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    for flags in (0, 1, 8):
        got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), (_cuda(ft[0]), _cuda(ft[1])),
                            (_cuda(fh[0]), _cuda(fh[1])), flags=flags).cpu().numpy()
        np.testing.assert_array_equal(got, want)
    if N == 1:
        assert (want == 0).all()


def test_rank_direction_flags_and_empty_filters():
    import oracle
    L = _lib()
    om, _ = gpu.synthetic_case("distmult", 300, 4, 64, seed=2)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(1)
    Q = 9
    qh, qr, qt = rng.randint(300, size=Q), rng.randint(4, size=Q), rng.randint(300, size=Q)
    want = oracle.rank_1vsall(om, qh, qr, qt)  # no filters: filtered == raw
    assert (want[:, 0] == want[:, 1]).all() and (want[:, 2] == want[:, 3]).all()
    tail = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), flags=L.RANK_TAIL_ONLY).cpu().numpy()
    head = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), flags=L.RANK_HEAD_ONLY).cpu().numpy()
    np.testing.assert_array_equal(tail[:, :2], want[:, :2]); assert (tail[:, 2:] == 0).all()
    np.testing.assert_array_equal(head[:, 2:], want[:, 2:]); assert (head[:, :2] == 0).all()
    # all-empty CSR filters (ptr of zeros) behave like no filters
    z = torch.zeros(Q + 1, dtype=torch.int64, device="cuda")
    e = torch.zeros(1, dtype=torch.int64, device="cuda")
    got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), (z, e[:0]), (z, e[:0])).cpu().numpy()
    np.testing.assert_array_equal(got, want)
    # too many queries for one call is an argument error, not a crash
    big = torch.zeros(70000, dtype=torch.int64, device="cuda")
    with pytest.raises(L.KgeError):
        L.rank_1vsall(desc, big, big, big)
    # profiled sweeps report how many directions their launch covered: the tensor-core sweep of a full call
    # covers both, the fp32 sweep of one direction covers one, also right after a tensor-core call
    om, _ = gpu.synthetic_case("distmult", 2000, 4, 64, seed=2)
    desc = gpu.desc_from_oracle_model(om)
    qh, qt = rng.randint(2000, size=Q), rng.randint(2000, size=Q)
    L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), flags=L.RANK_PROFILE)
    assert L.rank_last_sweep_directions() == 2
    L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), flags=L.RANK_PROFILE | L.RANK_NO_TC | L.RANK_TAIL_ONLY)
    assert L.rank_last_sweep_directions() == 1


def test_evaluator_batches_large_query_sets():
    """Evaluator.rank_triples splits > QUERY_BATCH queries into several kernel calls."""
    import oracle
    import pykg2vec_b200
    from pykg2vec_b200.evaluator import Evaluator
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    kg = SyntheticKnowledgeGraph(40, 3, 50, 5, 5, seed=0)
    cfg = SyntheticConfig(kg, hidden_size=8, l1_flag=True)
    torch.manual_seed(0)
    m = pykg2vec_b200.import_model("transe")(**cfg.__dict__).cuda()
    ev = Evaluator(m, cfg)
    ev.QUERY_BATCH = 500
    rng = np.random.RandomState(0)
    Q = 1203
    qh, qr, qt = rng.randint(40, size=Q), rng.randint(3, size=Q), rng.randint(40, size=Q)
    got = ev.rank_triples(qh, qr, qt)
    om = oracle.Model("transe", [w.detach().cpu().numpy() for w in m.kge_tables()], 8, l1_flag=True)
    np.testing.assert_array_equal(got, oracle.rank_1vsall(om, qh, qr, qt))


@pytest.mark.parametrize("name,d,l1", [("transh", 48, False), ("transh", 50, True), ("transd", 64, False),
                                       ("transd", 200, True)])
def test_relation_grouped_evaluation_equals_gather_sweep(name, d, l1):
    """TransH / TransD: projecting the entity table once per relation (kge_project_entities) and
    ranking that relation's queries with TransE's tiled sweep gives exactly the counts of the
    model's own (gather) sweep and of the oracle — including the reordering of queries and filters."""
    import types
    import oracle
    from pykg2vec_b200 import _lib
    from pykg2vec_b200.evaluator import Evaluator
    N, R, Q = 700, 5, 230
    om, tabs = gpu.synthetic_case(name, N, R, d, seed=d + len(name), l1=l1)
    desc = gpu.desc_from_oracle_model(om)
    # the projected table reproduces the model bit for bit through TransE
    rng = np.random.RandomState(4)
    h, t = rng.randint(N, size=64), rng.randint(N, size=64)
    for r in (0, R - 1):
        proj = _lib.project_entities(desc, r)
        te = _lib.ModelDesc("transe", [proj, desc.tables[1]], d, l1_flag=l1)
        rr = np.full(64, r, dtype=np.int64)
        ids = [torch.from_numpy(a).cuda() for a in (h, rr, t)]
        for grouping in (0, 1):
            a = _lib.score_fwd(te, *ids, grouping=grouping).cpu().numpy()
            b = _lib.score_fwd(desc, *ids, grouping=grouping).cpu().numpy()
            assert np.array_equal(gpu.bits(a), gpu.bits(b))
    # batched evaluator, queries of mixed relations in random order, with filters
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=9)
    model = types.SimpleNamespace(model_name=name, kge_desc=lambda: desc, kge_tables=lambda: desc.tables)
    ev = object.__new__(Evaluator)
    ev.model = model
    ev.config = types.SimpleNamespace(device="cuda", tot_entity=N, relation_grouped_eval=True, cuda_graph=False)
    ev._filter_cache, ev._workspace = {}, None
    got = ev.rank_triples(qh, qr, qt, ft, fh)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    assert np.array_equal(got, want)
    ev.config.relation_grouped_eval = False
    assert np.array_equal(ev.rank_triples(qh, qr, qt, ft, fh), want)
    ev.config.relation_grouped_eval = True
    assert np.array_equal(ev.rank_triples(qh, qr, qt)[:, 0], want[:, 0])     # no filters


def test_relation_grouped_evaluation_transr():
    import types
    import oracle
    from pykg2vec_b200.evaluator import Evaluator
    N, R, d, dr, Q = 500, 4, 24, 16, 160
    om, tabs = gpu.synthetic_case("transr", N, R, d, seed=11, dr=dr)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(4)
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=9)
    model = types.SimpleNamespace(model_name="transr", kge_desc=lambda: desc, kge_tables=lambda: desc.tables)
    ev = object.__new__(Evaluator)
    ev.model = model
    ev.config = types.SimpleNamespace(device="cuda", tot_entity=N, relation_grouped_eval=True, cuda_graph=False)
    ev._filter_cache, ev._workspace = {}, None
    assert np.array_equal(ev.rank_triples(qh, qr, qt, ft, fh), oracle.rank_1vsall(om, qh, qr, qt, ft, fh))


@pytest.mark.parametrize("name,d,l1", [("transe", 200, False), ("transe", 52, True), ("transm", 64, False), ("transe", 300, False)])
def test_score_fwd_large_batch_staged_kernel(name, d, l1, monkeypatch):
    """batches of >= 4 tiles per SM take the persistent cp.async-staged kernel (kge_score.cu): same bits as
    the register-cached kernel and the oracle, ragged last tile included, both groupings."""
    import oracle
    L = _lib()
    N, R = 3000, 11
    om, _ = gpu.synthetic_case(name, N, R, d, seed=d, l1=l1)
    desc = gpu.desc_from_oracle_model(om)
    n = 4 * torch.cuda.get_device_properties(0).multi_processor_count * 32 + 777
    rng = np.random.RandomState(1)
    h, r, t = rng.randint(N, size=n), rng.randint(R, size=n), rng.randint(N, size=n)
    for grouping in (0, 1):
        so = oracle.score_fwd(om, h, r, t, grouping)
        s = L.score_fwd(desc, _cuda(h), _cuda(r), _cuda(t), grouping).cpu().numpy()
        np.testing.assert_array_equal(gpu.bits(s), gpu.bits(so))
        monkeypatch.setenv("KGE_SCORE_NO_STAGED", "1")
        s2 = L.score_fwd(desc, _cuda(h), _cuda(r), _cuda(t), grouping).cpu().numpy()
        monkeypatch.delenv("KGE_SCORE_NO_STAGED")
        np.testing.assert_array_equal(gpu.bits(s2), gpu.bits(so))
