"""-m gpu tests of the tensor-core rank path around the sweep: the resolve-and-commit launch (band pairs, filter
corrections and the commit of the tensor-core counts in one launch per direction, or the fp32 tiled sweep when
the pair list overflows), the TransE fallback that stages the raw table and normalises it in shared memory, the
done counter across CUDA-graph replays, and workspaces of exactly kge_rank_workspace_bytes."""
import numpy as np
import pytest
import torch

import gpu_util as gpu

pytestmark = pytest.mark.gpu
TC_MODELS = ["transe", "distmult", "complex", "rotate", "cp", "rescal"]


def _lib():
    from pykg2vec_b200 import _lib
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _case(model, N, d, seed, degenerate=None, R=7):
    """oracle model + device description; degenerate: None, 'all' (every entity row identical: every pair
    ties, the band list overflows) or 'half' (every other row identical)."""
    import oracle
    L = _lib()
    margin = 6.0 if model == "rotate" else 0.0
    _, tabs = gpu.synthetic_case(model, N, R, d, seed=seed, margin=margin)
    ent_tables = {"transe": [0], "distmult": [0], "complex": [0, 1], "rotate": [0, 1], "cp": [0, 2], "rescal": [0]}[model]
    for k in ent_tables:
        if degenerate == "all":
            tabs[k][:] = tabs[k][0]
        elif degenerate == "half":
            tabs[k][::2] = tabs[k][0]
    om = oracle.Model(model, tabs, d, rel_dim=d, margin=margin,
                      embedding_range=(margin + 2.0) / d if model == "rotate" else None)
    desc = gpu.desc_from_oracle_model(om)
    if model == "rescal":   # Rescal.forward normalises its tables in place before scoring (pairwise.py:843-844)
        for t in desc.tables:
            L.normalize_rows(t)
        om = oracle.Model("rescal", [t.cpu().numpy() for t in desc.tables], d)
    return om, desc


def _queries(rng, N, R, Q):
    return rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)


@pytest.mark.parametrize("model", TC_MODELS)
@pytest.mark.parametrize("degenerate", ["all", "half"])
def test_overflow_fallback_ranks_exactly(model, degenerate):
    """Degenerate tables at N >= 1024 (the tensor-core path): with every entity row identical the pair list
    overflows and the resolve launch ranks the direction with the fp32 tiled sweep; with half of them identical
    it may or may not.  Counts equal the oracle's, with and without filters, and the fp32 path's."""
    import oracle
    L = _lib()
    N, d, Q = 1100, 64, 200
    om, desc = _case(model, N, d, seed=N + len(model), degenerate=degenerate)
    rng = np.random.RandomState(3)
    qh, qr, qt = _queries(rng, N, 7, Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=6)
    dft, dfh = (_cuda(ft[0]), _cuda(ft[1])), (_cuda(fh[0]), _cuda(fh[1]))
    for filt in (False, True):
        want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh) if filt else oracle.rank_1vsall(om, qh, qr, qt)
        if degenerate == "all" and not filt:
            assert (want == 0).all()
        for flags in (0, L.RANK_NO_TC, L.RANK_SINGLE_STREAM):
            args = (dft, dfh) if filt else (None, None)
            got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), *args, flags=flags).cpu().numpy()
            np.testing.assert_array_equal(got, want, err_msg="filters %s flags %d" % (filt, flags))


@pytest.mark.parametrize("layout", ["unaligned", "d_not_multiple_of_4"])
def test_transe_overflow_with_scratch_copy(layout):
    """TransE tables TMA cannot read directly (base not 16-byte aligned, or rows not whole 16-byte chunks)
    keep the normalised scratch copy for the fallback: both fallbacks rank exactly."""
    import oracle
    L = _lib()
    N, Q = 1024, 200
    d = 64 if layout == "unaligned" else 50
    om, _ = _case("transe", N, d, seed=9, degenerate="all")
    ent, rel = om.tables
    if layout == "unaligned":
        buf = torch.empty(N * d + 1, dtype=torch.float32, device="cuda")
        ent_dev = buf[1:].view(N, d)
        ent_dev.copy_(_cuda(ent))
        assert ent_dev.data_ptr() % 16 != 0
    else:
        ent_dev = _cuda(ent)
    desc = L.ModelDesc("transe", [ent_dev, _cuda(rel)], d)
    rng = np.random.RandomState(4)
    qh, qr, qt = _queries(rng, N, 7, Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=6)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), (_cuda(ft[0]), _cuda(ft[1])),
                        (_cuda(fh[0]), _cuda(fh[1]))).cpu().numpy()
    np.testing.assert_array_equal(got, want)


def test_graph_replays_equal_eager_calls():
    """The TransE rank call captured once as a CUDA graph and replayed with new tables, queries and filters
    copied into its static inputs, alternating inputs whose pair list overflows and inputs whose does not:
    every replay equals the eager call on the same inputs and the oracle (the resolve launch's done counter
    is reset for the next replay, and an overflowing replay leaves it as it found it)."""
    import oracle
    L = _lib()
    N, d, Q, R = 1536, 64, 200, 7
    rng = np.random.RandomState(12)
    cases = []
    for k, degenerate in enumerate([None, "all", None, "half", "all", None]):
        om, _ = _case("transe", N, d, seed=100 + k, degenerate=degenerate, R=R)
        qh, qr, qt = _queries(rng, N, R, Q)
        ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=4 + k)
        cases.append((om, qh, qr, qt, ft, fh))
    cap_t = max(c[4][1].size for c in cases)
    cap_h = max(c[5][1].size for c in cases)
    s_ent = torch.zeros((N, d), dtype=torch.float32, device="cuda")
    s_rel = torch.zeros((R, d), dtype=torch.float32, device="cuda")
    s_q = [torch.zeros(Q, dtype=torch.int64, device="cuda") for _ in range(3)]
    s_tp, s_hp = (torch.zeros(Q + 1, dtype=torch.int64, device="cuda") for _ in range(2))
    s_ti = torch.zeros(cap_t, dtype=torch.int64, device="cuda")
    s_hi = torch.zeros(cap_h, dtype=torch.int64, device="cuda")
    desc = L.ModelDesc("transe", [s_ent, s_rel], d)
    ws = torch.empty(L.rank_workspace_bytes(desc, Q), dtype=torch.uint8, device="cuda")
    counts = torch.zeros((Q, 4), dtype=torch.int32, device="cuda")

    def load(c):
        om, qh, qr, qt, ft, fh = c
        s_ent.copy_(_cuda(om.tables[0]))
        s_rel.copy_(_cuda(om.tables[1]))
        for s, a in zip(s_q, (qh, qr, qt)):
            s.copy_(_cuda(a))
        s_tp.copy_(_cuda(ft[0]))
        s_hp.copy_(_cuda(fh[0]))
        s_ti.zero_()
        s_hi.zero_()
        s_ti[:ft[1].size].copy_(_cuda(ft[1]))
        s_hi[:fh[1].size].copy_(_cuda(fh[1]))

    def body():
        counts.zero_()
        L.rank_1vsall(desc, *s_q, (s_tp, s_ti), (s_hp, s_hi), counts=counts, workspace=ws)

    load(cases[0])
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        body()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        body()
    for i, c in enumerate(cases):
        load(c)
        g.replay()
        torch.cuda.synchronize()
        got = counts.cpu().numpy().copy()
        eager = L.rank_1vsall(desc, *s_q, (s_tp, s_ti), (s_hp, s_hi), workspace=ws).cpu().numpy()
        om, qh, qr, qt, ft, fh = c
        want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
        np.testing.assert_array_equal(got, eager, err_msg="replay %d" % i)
        np.testing.assert_array_equal(got, want, err_msg="replay %d" % i)


@pytest.mark.parametrize("model", ["transe", "distmult", "cp"])
@pytest.mark.parametrize("Q", [1, 129, 512])
def test_exact_workspace_size(model, Q):
    """A workspace of exactly kge_rank_workspace_bytes holds every buffer of the call, with the pair list
    overflowing or not, at query counts below, across and at the width of a launch's query blocks: the call
    ranks exactly and writes nothing past the workspace's end."""
    import oracle
    L = _lib()
    N, d, guard = 1300, 64, 1 << 16
    for degenerate in (None, "all"):
        om, desc = _case(model, N, d, seed=Q, degenerate=degenerate)
        rng = np.random.RandomState(Q)
        qh, qr, qt = _queries(rng, N, 7, Q)
        ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=3)
        nbytes = L.rank_workspace_bytes(desc, Q)
        buf = torch.full((nbytes + guard,), 0xA5, dtype=torch.uint8, device="cuda")
        want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
        got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), (_cuda(ft[0]), _cuda(ft[1])),
                            (_cuda(fh[0]), _cuda(fh[1])), workspace=buf[:nbytes]).cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg="degenerate %s" % degenerate)
        assert (buf[nbytes:] == 0xA5).all().item(), "degenerate %s: write past the workspace" % degenerate
