"""-m gpu tests of the fused hinge + SGD training step (kge_train_pairwise_hinge_sgd) against the same step run
as a chain of independent kernels: score_fwd -> the hinge loss kernel -> score_bwd -> the dense SGD step.

The batches are built so that no embedding row receives more than two gradient contributions: a sum of at most
two floats onto a zero-filled scratch does not depend on the order of the atomics, so the updated tables must
be the same bits whichever way the step runs."""
import numpy as np
import pytest
import torch

import gpu_util as gpu

pytestmark = pytest.mark.gpu

# (model, d, dr, l1): the models of test_gpu_train.test_fused_hinge_sgd_matches_dense_sgd, TransE at the widths
# that select each register-cache depth of the step (d = 50 / 128 / 200), the looped form (d = 1000) and an odd
# width (scalar rows)
MODELS = [("transe", 200, None, False), ("transe", 50, None, True), ("transh", 48, None, False),
          ("transd", 40, None, True), ("transr", 25, 13, False), ("transm", 36, None, False),
          ("kg2e", 40, None, False), ("hole", 30, None, False), ("transe", 50, None, False),
          ("transe", 128, None, True), ("transe", 1000, None, False), ("transe", 33, None, False)]
BATCHES = [1, 7, 33, 512, 8192]
MARGIN, LR = 0.3, 0.05


def _batch(B, seed):
    """Each entity row in at most two triples (a head and its corrupted copy), each relation row in exactly one
    pair (the positive and its negative share it)."""
    rng = np.random.RandomState(seed)
    N, R = 3 * B + 5, B + 3
    e = rng.permutation(N)
    ph, pt, x = e[:B], e[B:2 * B], e[2 * B:3 * B]
    pr = rng.permutation(R)[:B]
    tail = rng.random_sample(B) > 0.5
    nh, nt = np.where(tail, ph, x), np.where(tail, x, pt)
    return N, R, [np.ascontiguousarray(a, dtype=np.int64) for a in (ph, pr, pt, nh, pr.copy(), nt)]


def _case(model, d, dr, l1, B):
    from pykg2vec_b200 import _lib
    N, R, ids = _batch(B, seed=B + d)
    om, _ = gpu.synthetic_case(model, N, R, d, seed=B + 7, dr=dr, l1=l1, scale=0.4)
    desc_f = gpu.desc_from_oracle_model(om)
    desc_c = gpu.desc_from_oracle_model(om)
    return _lib, om, desc_f, desc_c, [torch.from_numpy(a).cuda() for a in ids]


def _trained(model, k):
    return not (model == "transm" and k == 2)   # TransM's per-relation theta is not a parameter


def _chain_step(L, model, desc, ids):
    """score_fwd x2 -> hinge_kernel -> score_bwd x2 -> kge_optim_apply_dense (SGD) per trained table"""
    pos, neg = L.score_fwd(desc, *ids[:3]), L.score_fwd(desc, *ids[3:])
    loss, gp, gn = L.loss_pairwise_hinge(pos, neg, MARGIN)
    grads = [torch.zeros_like(t) for t in desc.tables]
    L.score_bwd(desc, *ids[:3], gp, grads)
    L.score_bwd(desc, *ids[3:], gn, grads)
    for k, (w, g) in enumerate(zip(desc.tables, grads)):
        if _trained(model, k):
            L.optim_apply_dense(w, g, L.OPT_SGD, LR)
    return pos, neg, loss


@pytest.mark.parametrize("B", BATCHES)
@pytest.mark.parametrize("spec", MODELS, ids=lambda s: "%s-d%d%s" % (s[0], s[1], "-l1" if s[3] else ""))
def test_fused_hinge_step_equals_the_kernel_chain(spec, B):
    model, d, dr, l1 = spec
    L, om, desc_f, desc_c, ids = _case(model, d, dr, l1, B)
    before = [t.cpu().numpy() for t in desc_f.tables]
    scratch = [torch.zeros_like(t) for t in desc_f.tables]
    loss = L.train_pairwise_hinge_sgd(desc_f, scratch, *ids, margin=MARGIN, lr=LR)
    pos, neg, _ = _chain_step(L, model, desc_c, ids)
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(zip(desc_f.tables, desc_c.tables)):
        assert np.array_equal(gpu.bits(a.cpu().numpy()), gpu.bits(b.cpu().numpy())), "%s B=%d table %d" % (model, B, k)
    assert all(float(s.abs().max()) == 0.0 for s in scratch), "gradient scratch must be left zeroed"
    # hinge activity: only entity rows of the pairs the score_fwd scores make active move (an active row may
    # still keep its bits where its gradient is zero or below half an ulp of the weight)
    sp, sn = pos.cpu().numpy(), neg.cpu().numpy()
    v = np.maximum((sp + np.float32(MARGIN)) - sn, np.float32(0))   # fp32 ops, as the kernels round them
    act = v > 0
    ent = [x.cpu().numpy() for x in ids]
    want = set(np.concatenate([ent[0][act], ent[2][act], ent[3][act], ent[5][act]]).tolist())
    moved = set(np.nonzero((desc_f.tables[0].cpu().numpy() != before[0]).any(axis=1))[0].tolist())
    assert moved <= want and (len(moved) > 0) == (len(want) > 0), "%s B=%d: %d rows moved, %d of active pairs" % (
        model, B, len(moved), len(want))
    # loss: the kernel's own hinge terms, summed in fp32 in some order, vs their fp64 sum
    ref = float(v.astype(np.float64).sum())
    assert abs(float(loss.item()) - ref) <= B * 2.0 ** -23 * ref + 1e-30, (float(loss.item()), ref)


@pytest.mark.parametrize("spec", [("transe", 200, None, False), ("transe", 1000, None, False), ("transr", 25, 13, False)],
                         ids=lambda s: "%s-d%d" % (s[0], s[1]))
def test_fused_hinge_step_graph_replay_equals_eager(spec):
    model, d, dr, l1 = spec
    B = 512
    L, om, desc_e, desc_g, ids = _case(model, d, dr, l1, B)
    s_e = [torch.zeros_like(t) for t in desc_e.tables]
    s_g = [torch.zeros_like(t) for t in desc_g.tables]
    loss_e = L.train_pairwise_hinge_sgd(desc_e, s_e, *ids, margin=MARGIN, lr=LR)
    loss_g = torch.zeros(1, dtype=torch.float32, device="cuda")
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):   # un-captured warm-up with lr = 0: the tables stay as they are
        L.train_pairwise_hinge_sgd(desc_g, s_g, *ids, margin=MARGIN, lr=0.0, loss_out=loss_g)
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        L.train_pairwise_hinge_sgd(desc_g, s_g, *ids, margin=MARGIN, lr=LR, loss_out=loss_g)
    g.replay()
    torch.cuda.synchronize()
    for k, (a, b) in enumerate(zip(desc_e.tables, desc_g.tables)):
        assert np.array_equal(gpu.bits(a.cpu().numpy()), gpu.bits(b.cpu().numpy())), "table %d" % k
    assert all(float(s.abs().max()) == 0.0 for s in s_g)
    assert abs(float(loss_g.item()) - float(loss_e.item())) <= B * 2.0 ** -23 * abs(float(loss_e.item()))
