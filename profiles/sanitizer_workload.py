"""Workload for compute-sanitizer (memcheck / racecheck / synccheck): every kernel with hand-rolled
cross-warp synchronisation or atomics, at small sizes — the tensor-core sweep (TMA + mbarrier +
wgmma), the fp32 tiled sweep (TMA + mbarrier + release counters; whole-row and slab mode, all OPs), the
exact-resolve kernel, the fp32 sweep's commit-or-fallback entry, the fused hinge step (atom.exch sparse apply), the
fused RotatE self-adversarial step (warp team and CTA team) and the dense optimizer.  Results are checked against the oracle so a silent corruption would also fail here.

    compute-sanitizer --tool memcheck  python profiles/sanitizer_workload.py
    compute-sanitizer --tool racecheck python profiles/sanitizer_workload.py
"""
import os, sys
import numpy as np, torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__))); sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import gpu_util as gpu
import oracle
from pykg2vec_b200 import _lib
cu = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
small = os.environ.get("KGE_SANITIZER_SMALL") == "1"
cases = [("transe", 1300, 200, 0.0), ("distmult", 1200, 36, 0.0), ("complex", 1100, 52, 0.0), ("rotate", 1100, 40, 6.0),
         ("cp", 1200, 40, 0.0), ("rescal", 1100, 16, 0.0), ("rotate", 1100, 600 if not small else 300, 12.0), ("hole", 300, 32, 0.0),
         ("simple", 400, 48, 0.0), ("transm", 300, 64, 0.0)]
for name, N, d, margin in cases:
    om, _ = gpu.synthetic_case(name, N, 5, d, seed=N + d, margin=margin)
    desc = gpu.desc_from_oracle_model(om)
    if name == "rescal":
        for t in desc.tables: _lib.normalize_rows(t)
        om = oracle.Model("rescal", [t.cpu().numpy() for t in desc.tables], d)
    rng = np.random.RandomState(d)
    Q = 70
    qh, qr, qt = rng.randint(N, size=Q), rng.randint(5, size=Q), rng.randint(N, size=Q)
    ft, fh = gpu.random_filters_csr(rng, N, qh, qr, qt, per_query=4)
    want = oracle.rank_1vsall(om, qh, qr, qt, ft, fh)
    for flags in (0, _lib.RANK_NO_TC):
        got = _lib.rank_1vsall(desc, cu(qh), cu(qr), cu(qt), (cu(ft[0]), cu(ft[1])), (cu(fh[0]), cu(fh[1])), flags=flags).cpu().numpy()
        assert np.array_equal(got, want), (name, flags)
    print("rank ok", name, N, d, flush=True)
# degenerate table -> list overflow -> on-device fallback
om, tabs = gpu.synthetic_case("distmult", 2048, 3, 32, seed=1)
tabs[0][:] = tabs[0][0]
om = oracle.Model("distmult", tabs, 32)
desc = gpu.desc_from_oracle_model(om)
rng = np.random.RandomState(0)
qh, qr, qt = rng.randint(2048, size=150), rng.randint(3, size=150), rng.randint(2048, size=150)
assert np.array_equal(_lib.rank_1vsall(desc, cu(qh), cu(qr), cu(qt)).cpu().numpy(), oracle.rank_1vsall(om, qh, qr, qt))
print("overflow fallback ok", flush=True)
# fused hinge + sparse apply, dense optimizer
om, tabs = gpu.synthetic_case("transe", 500, 7, 64, seed=3)
desc = gpu.desc_from_oracle_model(om)
scratch = [torch.zeros_like(t) for t in desc.tables]
ids = [cu(rng.randint(500 if k % 3 != 1 else 7, size=256)) for k in range(6)]
for _ in range(3):
    _lib.train_pairwise_hinge_sgd(desc, scratch, *ids, margin=1.0, lr=0.01)
assert all(float(s.abs().max()) == 0.0 for s in scratch)
g = torch.randn_like(desc.tables[0]); m1 = torch.zeros_like(g); m2 = torch.zeros_like(g)
for opt in (0, 1, 2):
    gg = g.clone()
    _lib.optim_apply_dense(desc.tables[0], gg, opt, 0.01, m1, m2, step=1)
    assert float(gg.abs().max()) == 0.0
# fused RotatE self-adversarial step: warp team (neg_rate <= 4) and CTA team
om, tabs = gpu.synthetic_case("rotate", 400, 5, 48, seed=9, margin=6.0)
desc = gpu.desc_from_oracle_model(om)
for neg_rate, B in ((2, 37), (24, 19)):
    ids = [cu(rng.randint(400 if k % 3 != 1 else 5, size=B if k < 3 else B * neg_rate)) for k in range(6)]
    gs = [torch.zeros_like(t) for t in desc.tables]
    loss = _lib.train_pairwise_selfadv(desc, gs, *ids, neg_rate=neg_rate, alpha=0.5)
    pos, neg = _lib.score_fwd(desc, *ids[:3]), _lib.score_fwd(desc, *ids[3:])
    want, _gp, _gn = _lib.loss_selfadv(pos, neg, neg_rate, 0.5)
    assert abs(loss.item() - want.item()) <= 1e-5 * abs(want.item())
torch.cuda.synchronize()
print("train ok", flush=True)
