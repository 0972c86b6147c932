"""-m gpu parity tests AT THE BASELINE.json SHAPES (N = 14,541 / 40,943 / 14,951 / 123,182; Q = 512,
the benched launch geometry): the CUDA path through the C-ABI vs
  * the CPU oracle — rank counts identical, flat scores bit-identical; all three sweep
    implementations (tensor-core two-level, fp32 tiled, gather) where they exist;
  * the reference itself (tests/golden/shapes_*.npz, written by make_golden_shapes.py from the
    UNMODIFIED reference on tables regenerated from the same seed): scores within 1e-4 relative,
    ranks identical on every query whose rank is well defined in fp32 (a float64 evaluation brackets
    the rank any fp32 summation order can report; outside that bracket nothing may fall).
Plus the size-independent properties of the sweep at these shapes: partial counts of row shards
add up, exact ties are never counted as better, a degenerate table (list overflow) still ranks
exactly through the on-device fallback."""
import json
import os

import numpy as np
import pytest
import torch

import golden_util as gu
import gpu_util as gpu

pytestmark = pytest.mark.gpu
Q_BENCH = 512
# queries checked against the (OpenMP, scalar C) oracle per case: the kernels always run all 512
ORACLE_QUERIES = {"cfg2_transe_fb15k237": 512, "cfg3_distmult_wn18rr": 192, "cfg3_complex_wn18rr": 128,
                  "cfg4_rotate_fb15k": 96, "cfg5_complex_yago310": 48}


def _lib():
    from pykg2vec_b200 import _lib
    return _lib


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _desc(spec, tables):
    L = _lib()
    phase = float(np.float32(np.pi / ((spec["margin"] + 2.0) / spec["d"]))) if spec["model"] == "rotate" else 0.0
    return L.ModelDesc(spec["model"], [_cuda(t) for t in tables], spec["d"], l1_flag=spec["l1"],
                       margin=spec["margin"], phase_scale=phase)


def _record(name, payload):
    """measured facts (band sizes, tensor-core error) as JSON under $KGE_TEST_RECORD_DIR, when it is set"""
    out = os.environ.get("KGE_TEST_RECORD_DIR")
    if not out:
        return
    os.makedirs(out, exist_ok=True)
    with open(os.path.join(out, "tc_parity_%s.json" % name), "w") as f:
        json.dump(payload, f)


@pytest.mark.parametrize("name", list(gu.BASELINE_SHAPES))
def test_baseline_shape_parity(name):
    import oracle
    L = _lib()
    spec = gu.BASELINE_SHAPES[name]
    tables = gu.baseline_tables(spec)
    g = dict(np.load(gu.shape_case_path(name)))
    np.testing.assert_array_equal(tables[0][:2, :8], g["table0_head"])   # same tables as the generator's
    om = gu.baseline_oracle_model(spec, tables)
    desc = _desc(spec, tables)
    N, R = spec["N"], spec["R"]

    # flat scores: bit-equal to the oracle, <= 1e-4 relative to the reference
    for grouping in (0, 1):
        s = L.score_fwd(desc, _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"]), grouping).cpu().numpy()
        np.testing.assert_array_equal(gpu.bits(s), gpu.bits(oracle.score_fwd(om, g["h"], g["r"], g["t"], grouping)))
    s = L.score_fwd(desc, _cuda(g["h"]), _cuda(g["r"]), _cuda(g["t"])).cpu().numpy()
    ref = g["scores"]
    err = np.abs(s.astype(np.float64) - ref) / np.maximum(np.abs(ref), 1e-2 * np.abs(ref).max())
    assert err.max() < 1e-4, (name, err.max())

    # Q = 512 queries with filters: the first ones are the reference's golden queries
    rng = np.random.RandomState(spec["seed"] + 2)
    nq = g["ranks"].shape[0]
    qh = np.concatenate([g["h"][:nq], rng.randint(N, size=Q_BENCH - nq)])
    qr = np.concatenate([g["r"][:nq], rng.randint(R, size=Q_BENCH - nq)])
    qt = np.concatenate([g["t"][:nq], rng.randint(N, size=Q_BENCH - nq)])
    ft, fh = gpu.random_filters_csr(rng, N, qh[nq:], qr[nq:], qt[nq:], per_query=10)
    ft = (np.concatenate([g["filt_t_ptr"], g["filt_t_ptr"][-1] + ft[0][1:]]), np.concatenate([g["filt_t_idx"], ft[1]]))
    fh = (np.concatenate([g["filt_h_ptr"], g["filt_h_ptr"][-1] + fh[0][1:]]), np.concatenate([g["filt_h_idx"], fh[1]]))
    dev = [_cuda(x) for x in (qh, qr, qt)]
    dft, dfh = (_cuda(ft[0]), _cuda(ft[1])), (_cuda(fh[0]), _cuda(fh[1]))
    got_tc = L.rank_1vsall(desc, *dev, dft, dfh).cpu().numpy()                        # tensor-core two-level
    got_fp32 = L.rank_1vsall(desc, *dev, dft, dfh, flags=L.RANK_NO_TC).cpu().numpy()  # fp32 tiled sweep
    np.testing.assert_array_equal(got_tc, got_fp32)

    # vs the oracle on a prefix of the queries (the oracle is scalar C)
    no = ORACLE_QUERIES[name]
    fto = (ft[0][:no + 1], ft[1][:ft[0][no]])
    fho = (fh[0][:no + 1], fh[1][:fh[0][no]])
    want = oracle.rank_1vsall(om, qh[:no], qr[:no], qt[:no], fto, fho)
    np.testing.assert_array_equal(got_tc[:no], want)
    # gather sweep on a few queries (it is 10x slower and only a cross-check here)
    ng = 16
    got_g = L.rank_1vsall(desc, *[x[:ng].contiguous() for x in dev], (_cuda(ft[0][:ng + 1]), _cuda(ft[1][:ft[0][ng]])),
                          (_cuda(fh[0][:ng + 1]), _cuda(fh[1][:fh[0][ng]])), flags=L.RANK_FORCE_GATHER).cpu().numpy()
    np.testing.assert_array_equal(got_g, want[:ng])

    # vs the reference's own ranks: identical wherever fp32 defines the rank, inside the fp64 bracket otherwise
    ambiguous = 0
    for i in range(nq):
        for direction, col in ((0, 0), (1, 2)):
            s64 = gu.fp64_candidate_scores(spec, tables, int(qh[i]), int(qr[i]), int(qt[i]), direction)
            tgt = int(qt[i]) if direction == 0 else int(qh[i])
            lo, hi = gu.rank_interval(s64, tgt)
            assert lo <= int(g["ranks"][i, col]) <= hi, (name, i, direction, "reference outside its own fp64 bracket")
            assert lo <= int(got_tc[i, col]) <= hi, (name, i, direction, lo, hi, int(got_tc[i, col]))
            if lo == hi:
                assert int(got_tc[i, col]) == int(g["ranks"][i, col])
                # the filtered rank subtracts well-defined filter entries only when they are unambiguous too
            else:
                ambiguous += 1
    exact = int((got_tc[:nq] == g["ranks"]).all(axis=1).sum())
    _record(name, {"case": name, "golden_queries": int(nq), "queries_identical_to_reference": exact,
                   "ambiguous_directions_fp64": ambiguous, "oracle_queries": int(no), "score_rel_err_max": float(err.max())})


def _band(dots, band):
    """(certainly better, certainly not) masks of level 1 from the probe's band description."""
    coef, cn = band
    coef, cn = coef.cpu().numpy().astype(np.float64), cn.cpu().numpy().astype(np.float64)
    half = coef[:, 1:2] + coef[:, 2:3] * cn[None, :] + coef[:, 3:4] * cn[None, :] ** 2
    u = dots.astype(np.float64) - coef[:, 0:1]
    return u > half, u < -half, half


@pytest.mark.parametrize("name", ["cfg2_transe_fb15k237", "cfg3_distmult_wn18rr", "cfg3_complex_wn18rr",
                                  "cfg4_rotate_fb15k"])
def test_tensor_core_level_is_consistent_with_exact_scores(name):
    """Level 1 alone: every candidate the tensor-core pass calls 'certainly better' / 'certainly not'
    must be so in the canonical fp32 scores, and the measured |D_tc - D_fp64| must sit well inside the
    proven bound used for the band (DESIGN.md §4b)."""
    import oracle
    L = _lib()
    spec = gu.BASELINE_SHAPES[name]
    tables = gu.baseline_tables(spec)
    om = gu.baseline_oracle_model(spec, tables)
    desc = _desc(spec, tables)
    N, R = spec["N"], spec["R"]
    rng = np.random.RandomState(7)
    Q = 160   # not a multiple of the 128-query block
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    stats = {"case": name, "Q": Q, "N": N}
    for direction in (0, 1):
        dots, band_desc, counts = L.rank_tc_probe(desc, _cuda(qh), _cuda(qr), _cuda(qt), direction)
        dots, counts = dots.cpu().numpy(), counts.cpu().numpy()
        yes, no, half = _band(dots, band_desc)
        want = oracle.rank_1vsall(om, qh, qr, qt)
        col = 0 if direction == 0 else 2
        np.testing.assert_array_equal(counts[:, col], want[:, col])
        band = 0
        max_ratio = 0.0
        for i in range(0, Q, 8):   # exact classification check on a sample of the queries
            cand = np.arange(N)
            if direction == 0:
                s = oracle.score_fwd(om, np.full(N, qh[i]), np.full(N, qr[i]), cand, 0)
                thr = oracle.score_fwd(om, qh[i:i + 1], qr[i:i + 1], qt[i:i + 1], 0)[0]
            else:
                s = oracle.score_fwd(om, cand, np.full(N, qr[i]), np.full(N, qt[i]), 1)
                thr = oracle.score_fwd(om, qh[i:i + 1], qr[i:i + 1], qt[i:i + 1], 1)[0]
            better = s < thr
            sure_yes, sure_no = yes[i], no[i]
            assert better[sure_yes].all(), (name, direction, i)
            assert (~better[sure_no]).all(), (name, direction, i)
            band += int((~sure_yes & ~sure_no).sum())
            # measured tensor-core error against float64 on the same decision quantity: the accumulator is an
            # affine function of the exact score; fit it on the fp64 scores and look at the residual
            s64 = gu.fp64_candidate_scores(spec, tables, int(qh[i]), int(qr[i]), int(qt[i]), direction)
            y = s64 if spec["model"] in ("distmult",) else (s64 * s64 if spec["model"] == "transe" else s64)
            A = np.vstack([y, np.ones_like(y)]).T
            coef, *_ = np.linalg.lstsq(A, dots[i].astype(np.float64), rcond=None)
            resid = np.abs(A @ coef - dots[i])
            max_ratio = max(max_ratio, float((resid / np.maximum(half[i], 1e-30)).max()))
        stats["dir%d" % direction] = {"band_pairs_per_query": band / len(range(0, Q, 8)),
                                      "max_residual_over_half_band": max_ratio}
        assert max_ratio < 0.5, (name, direction, max_ratio)   # the proven bound has >= 2x headroom on real data
    _record("probe_" + name, stats)


@pytest.mark.parametrize("model", ["complex", "distmult", "rotate"])
def test_heavy_rows_do_not_widen_every_band(model):
    """Trained tables hold rows far heavier than the typical one (Adagrad moves every touched element by ~lr per
    step).  The band of a pair scales with THAT candidate's norm, so a heavy sub-population must neither change
    the counts nor push the light candidates into the band (with one global max|c| the list overflowed and the
    fp32 sweep re-did the direction: 1.15 ms instead of 0.3 ms for ComplEx at the WN18RR shape)."""
    import oracle
    L = _lib()
    spec = dict(model=model, N=20000, R=11, d=200, l1=False, margin=6.0 if model == "rotate" else 0.0, seed=5)
    tables = gu.baseline_tables(spec)
    rng = np.random.RandomState(11)
    heavy = rng.choice(spec["N"], size=spec["N"] // 4, replace=False)
    for tix, kind in enumerate(gu._SHAPE_TABLES[model]):
        if kind == "e":
            tables[tix][heavy] *= 8.0
    om = gu.baseline_oracle_model(spec, tables)
    desc = _desc(spec, tables)
    Q = 128
    qh, qr, qt = rng.randint(spec["N"], size=Q), rng.randint(spec["R"], size=Q), rng.randint(spec["N"], size=Q)
    want = oracle.rank_1vsall(om, qh, qr, qt)
    got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt)).cpu().numpy()
    np.testing.assert_array_equal(got, want)
    for direction in (0, 1):
        dots, band_desc, _ = L.rank_tc_probe(desc, _cuda(qh), _cuda(qr), _cuda(qt), direction)
        yes, no, _half = _band(dots.cpu().numpy(), band_desc)
        per_query = float((~yes & ~no).sum()) / Q
        assert per_query < 128, (model, direction, per_query)   # the list holds 512 per query


def test_exact_ties_are_never_better():
    """duplicated entity rows (exact score ties with the target, and with each other): every sweep
    and the oracle count a tie as 'not better' — DESIGN.md §3."""
    import oracle
    L = _lib()
    for model, d in (("transe", 200), ("distmult", 200), ("complex", 100), ("rotate", 64)):
        spec = dict(model=model, N=3000, R=7, d=d, l1=False, margin=6.0 if model == "rotate" else 0.0, seed=99)
        tables = gu.baseline_tables(spec)
        rng = np.random.RandomState(3)
        # 40 groups of 25 identical entities
        for k in range(40):
            rows = rng.choice(spec["N"], size=25, replace=False)
            for tix, kind in enumerate(gu._SHAPE_TABLES[model]):
                if kind == "e":
                    tables[tix][rows] = tables[tix][rows[0]]
            if k == 0:
                dup = rows
        om = gu.baseline_oracle_model(spec, tables)
        desc = _desc(spec, tables)
        Q = 300
        qh, qr, qt = rng.randint(spec["N"], size=Q), rng.randint(spec["R"], size=Q), rng.randint(spec["N"], size=Q)
        qt[:25], qh[25:50] = dup, dup   # targets inside a duplicate group
        want = oracle.rank_1vsall(om, qh, qr, qt)
        for flags in (0, L.RANK_NO_TC, L.RANK_FORCE_GATHER):
            got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), flags=flags).cpu().numpy()
            np.testing.assert_array_equal(got, want, err_msg="%s flags %d" % (model, flags))


def test_degenerate_table_overflows_to_the_exact_sweep():
    """every entity identical -> every pair is a tie -> every pair lands in the band, the pair list
    overflows and the device-side fallback (fp32 tiled sweep) must produce the counts: all zero."""
    import oracle
    L = _lib()
    spec = dict(model="distmult", N=4096, R=3, d=64, l1=False, margin=0.0, seed=5)
    tables = gu.baseline_tables(spec)
    tables[0][:] = tables[0][0]
    om = gu.baseline_oracle_model(spec, tables)
    desc = _desc(spec, tables)
    rng = np.random.RandomState(1)
    Q = 200
    qh, qr, qt = rng.randint(spec["N"], size=Q), rng.randint(spec["R"], size=Q), rng.randint(spec["N"], size=Q)
    want = oracle.rank_1vsall(om, qh, qr, qt)
    assert (want == 0).all()
    got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt)).cpu().numpy()
    np.testing.assert_array_equal(got, want)
    # and a table that is degenerate only in part: half the rows identical, half random
    tables = gu.baseline_tables(spec)
    tables[0][::2] = tables[0][0]
    om = gu.baseline_oracle_model(spec, tables)
    desc = _desc(spec, tables)
    want = oracle.rank_1vsall(om, qh, qr, qt)
    got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt)).cpu().numpy()
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("model,N,d,Q", [("transe", 1024, 200, 130), ("distmult", 1100, 36, 257), ("complex", 1500, 52, 64),
                                         ("rotate", 2049, 200, 129), ("cp", 1300, 40, 100), ("rescal", 1200, 24, 77)])
def test_tensor_core_sweep_ragged_geometries(model, N, d, Q):
    """tile / query-block / k-block raggedness of the tensor-core sweep: N not a multiple of 128, Q not a
    multiple of 128, K not a multiple of 64 (and of 16; the last k-block is a zero-filled TMA tile), the
    streamed-query mode (K > 256)."""
    import oracle
    L = _lib()
    om, _ = gpu.synthetic_case(model, N, 5, d, seed=N + d, margin=6.0 if model == "rotate" else 0.0)
    desc = gpu.desc_from_oracle_model(om)
    rng = np.random.RandomState(d)
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(5, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=5)
    if model == "rescal":   # Rescal.forward normalises its tables in place before scoring (pairwise.py:843-844)
        for t in desc.tables:
            L.normalize_rows(t)
        om = oracle.Model("rescal", [t.cpu().numpy() for t in desc.tables], d)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    for flags in (0, L.RANK_NO_TC, 8):
        got = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), (_cuda(ft[0]), _cuda(ft[1])),
                            (_cuda(fh[0]), _cuda(fh[1])), flags=flags).cpu().numpy()
        np.testing.assert_array_equal(got, want, err_msg="flags %d" % flags)


def test_config5_row_shards_on_one_gpu():
    """configs[4]: ComplEx YAGO3-10 shape row-partitioned 8 ways (15,398 rows per shard), every shard
    swept separately with the compact query table — partial counts add up to the replicated result."""
    import oracle
    L = _lib()
    spec = gu.BASELINE_SHAPES["cfg5_complex_yago310"]
    tables = gu.baseline_tables(spec)
    desc = _desc(spec, tables)
    N, R, d = spec["N"], spec["R"], spec["d"]
    rng = np.random.RandomState(11)
    Q = Q_BENCH
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=8)
    dft, dfh = (_cuda(ft[0]), _cuda(ft[1])), (_cuda(fh[0]), _cuda(fh[1]))
    full = L.rank_1vsall(desc, _cuda(qh), _cuda(qr), _cuda(qt), dft, dfh).cpu().numpy()
    uniq = np.unique(np.concatenate([qh, qt]))
    remap = np.zeros(N, dtype=np.int64)
    remap[uniq] = np.arange(len(uniq))
    qtabs = [_cuda(tables[0][uniq]), _cuda(tables[1][uniq]), desc.tables[2], desc.tables[3]]
    qdesc = L.ModelDesc("complex", qtabs, d)
    counts = torch.zeros((Q, 4), dtype=torch.int32, device="cuda")
    per = (N + 7) // 8
    for g in range(8):
        lo, hi = g * per, min(N, (g + 1) * per)
        stabs = [desc.tables[0][lo:hi].contiguous(), desc.tables[1][lo:hi].contiguous(), desc.tables[2], desc.tables[3]]
        sdesc = L.ModelDesc("complex", stabs, d)
        L.rank_1vsall(sdesc, _cuda(remap[qh]), _cuda(qr), _cuda(remap[qt]), dft, dfh, counts=counts, row_lo=lo, row_hi=hi,
                      query_desc=qdesc, tgt_h=_cuda(qh), tgt_t=_cuda(qt))
    np.testing.assert_array_equal(counts.cpu().numpy(), full)
    om = gu.baseline_oracle_model(spec, tables)
    no = 24
    want = oracle.rank_1vsall(om, qh[:no], qr[:no], qt[:no], (ft[0][:no + 1], ft[1][:ft[0][no]]), (fh[0][:no + 1], fh[1][:fh[0][no]]))
    np.testing.assert_array_equal(full[:no], want)
