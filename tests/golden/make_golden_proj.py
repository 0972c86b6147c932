#!/usr/bin/env python
"""Golden fixtures for the projection-model tail (SURVEY.md §8 row a11 / f4) by RUNNING THE
REFERENCE's ConvE (pykg2vec/models/projection.py:12-125) and Criterion.multi_class_bce
(pykg2vec/utils/criterion.py:41-50) on seeded inputs, torch CPU fp32.

Run in the build container only (needs /root/reference):
    python tests/golden/make_golden_proj.py

Per case (conve_*.npz):
  sd_<key>            the reference model's full state_dict (parameters and BN buffers)
  h, r, t             triple ids [b]
  x_tail / x_head     eval-mode trunk output [b,k] — the operand of `x . E^T + b`
                      (projection.py:88-99 re-evaluated with the reference's own sub-modules; the
                      script asserts sigmoid(x E^T + b) == model.forward bit for bit)
  preds_tail / _head  eval-mode model.forward(e, r, direction) [b,N]
  tr_* (train mode, dropouts 0): x, preds, dense labels hr_t / tr_h, the loss of
                      Criterion.multi_class_bce with label smoothing 0.1, and autograd gradients of
                      every parameter (grad_<key>), plus d loss / d x_tail, d loss / d x_head
  ranks               (trank, ftrank, hrank, fhrank) from the reference Evaluator.test_*_rank ->
                      model.predict_*_rank -> MetricCalculator.get_*_rank walk, with the filters
"""
import copy
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the import stubs and /root/reference on sys.path)

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402

CASES = [
    # name, N, R, hidden_size, hidden_size_1, b
    ("conve_d48", 97, 5, 48, 8, 24),
    ("conve_d100", 211, 7, 100, 10, 20),
]
N_QUERIES = 6
LABEL_SMOOTHING = 0.1
GRAD_SAMPLE_STRIDE = 37


def trunk(m, e, r):
    """ConvE.forward + inner_forward up to (not including) the x.E^T product, using the
    reference's own sub-modules (projection.py:104-112 and :88-99)."""
    e_emb, r_emb = m.embed2(e, r)
    stacked_e = e_emb.view(-1, 1, m.hidden_size_2, m.hidden_size_1)
    stacked_r = r_emb.view(-1, 1, m.hidden_size_2, m.hidden_size_1)
    x = torch.cat([stacked_e, stacked_r], 2)
    x = m.bn0(x)
    x = m.inp_drop(x)
    x = m.conv2d_1(x)
    x = m.bn1(x)
    x = torch.relu(x)
    x = m.feat_drop(x)
    x = x.view(e.shape[0], -1)
    x = m.fc(x)
    x = m.hidden_drop(x)
    if m.training:
        x = m.bn2(x)
    return torch.relu(x)


def make_case(name, N, R, k, k1, b, seed):
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1000)
    m = ref_projection.ConvE(tot_entity=N, tot_relation=R, hidden_size=k, hidden_size_1=k1, lmbda=0.1,
                             input_dropout=0.0, feature_map_dropout=0.0, hidden_dropout=0.0)
    with torch.no_grad():
        # the reference leaves nn.Embedding's N(0,1) initialisation; make BN / bias non-trivial
        m.ent_embeddings.weight.mul_(0.5)
        m.rel_embeddings.weight.mul_(0.5)
        m.b.weight.normal_(0.0, 0.3)
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.6, 1.4)
            bn.bias.normal_(0.0, 0.2)
            bn.running_mean.normal_(0.0, 0.2)
            bn.running_var.uniform_(0.5, 1.5)
    out = {"N": N, "R": R, "hidden_size": k, "hidden_size_1": k1, "label_smoothing": np.float32(LABEL_SMOOTHING)}
    for key, v in m.state_dict().items():
        out["sd_" + key] = v.detach().numpy().copy()
    h = rng.randint(N, size=b).astype(np.int64)
    r = rng.randint(R, size=b).astype(np.int64)
    t = rng.randint(N, size=b).astype(np.int64)
    ht, rt, tt = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)
    out.update(h=h, r=r, t=t)

    # ---- eval mode ---------------------------------------------------------------------------
    m.eval()
    with torch.no_grad():
        x_tail = trunk(m, ht, rt)
        x_head = trunk(m, tt, rt + R)
        p_tail = m.forward(ht, rt, direction="tail")
        p_head = m.forward(tt, rt, direction="head")
        for x, p in ((x_tail, p_tail), (x_head, p_head)):
            again = torch.sigmoid(torch.add(torch.matmul(x, m.ent_embeddings.weight.T), m.b.weight))
            assert torch.equal(again, p), "trunk() is not what the reference forward evaluates"
    out.update(x_tail=x_tail.numpy().copy(), x_head=x_head.numpy().copy(),
               preds_tail=p_tail.numpy().copy(), preds_head=p_head.numpy().copy())
    q = [(int(h[i]), int(r[i]), int(t[i])) for i in range(N_QUERIES)]
    hr_t, tr_h = mg.random_filters(rng, N, R, q)
    out["ranks"] = mg.reference_ranks(m, N, q, hr_t, tr_h)
    out["filt_t_ptr"], out["filt_t_idx"] = mg.csr(hr_t, [(a, b_) for a, b_, c in q])
    out["filt_h_ptr"], out["filt_h_idx"] = mg.csr(tr_h, [(c, b_) for a, b_, c in q])

    # ---- train mode: trainer.py:159-166 (train_step_projection) + criterion.py:41-50 -----------
    mt = copy.deepcopy(m)
    mt.train()
    lab_t = (rng.rand(b, N) < 0.03).astype(np.float32)   # hr_t rows as generator.py:180-196 builds them
    lab_h = (rng.rand(b, N) < 0.03).astype(np.float32)
    lab_t[np.arange(b), t] = 1.0
    lab_h[np.arange(b), h] = 1.0
    mt.zero_grad()
    xt = trunk(copy.deepcopy(mt), ht, rt)            # a copy: BN running stats must not advance twice
    xh = trunk(copy.deepcopy(mt), tt, rt + R)
    pred_tails = mt(ht, rt, direction="tail")
    pred_heads = mt(tt, rt, direction="head")
    loss = Criterion.multi_class_bce(pred_heads, pred_tails, torch.from_numpy(lab_h), torch.from_numpy(lab_t),
                                     LABEL_SMOOTHING, N)
    loss.backward()
    out.update(tr_x_tail=xt.detach().numpy().copy(), tr_x_head=xh.detach().numpy().copy(),
               tr_preds_tail=pred_tails.detach().numpy().copy(), tr_preds_head=pred_heads.detach().numpy().copy(),
               tr_labels_tail=lab_t, tr_labels_head=lab_h, tr_loss=np.float32(loss.item()))
    for key, p in mt.named_parameters():
        g = p.grad.detach().numpy().copy()
        if g.size > 200000:   # keep the fixture small: a strided sample of the large fc.weight gradient
            out["gradsample_" + key] = g.reshape(-1)[::GRAD_SAMPLE_STRIDE].copy()
        else:
            out["grad_" + key] = g
    for key, v in mt.state_dict().items():   # BN running statistics after the two training forwards
        if "running" in key:
            out["sd_after_" + key] = v.detach().numpy().copy()
    # gradient w.r.t. the tail operand x and the dense preds (checks of the tail kernels alone)
    for tag, x, lab in (("tail", xt, lab_t), ("head", xh, lab_h)):
        xd = x.detach().clone().requires_grad_()
        E = mt.ent_embeddings.weight.detach().clone().requires_grad_()
        bb = mt.b.weight.detach().clone().requires_grad_()
        p = torch.sigmoid(torch.add(torch.matmul(xd, E.T), bb))
        y = torch.from_numpy(lab) * (1.0 - LABEL_SMOOTHING) + 1.0 / N
        one = torch.mean(torch.nn.BCEWithLogitsLoss()(p, y))
        one.backward()
        out["tr_loss_" + tag] = np.float32(one.item())
        out["tr_gx_" + tag] = xd.grad.numpy().copy()
        out["tr_gE_" + tag] = E.grad.numpy().copy()
        out["tr_gb_" + tag] = bb.grad.numpy().copy()
    # arrays over 1 MB (the d=100 fc.weight) go to golden/split/ in two row blocks (golden_util.load joins them)
    big = {k: out.pop(k) for k in list(out) if getattr(out[k], "nbytes", 0) > (1 << 20)}
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    for k, v in big.items():
        os.makedirs(os.path.join(HERE, "split"), exist_ok=True)
        for part, rows in enumerate(np.array_split(v, 2)):
            np.savez_compressed(os.path.join(HERE, "split", "%s.%d.npz" % (name, part)), **{k: rows})
    print("wrote", name, "loss", out["tr_loss"], "ranks[0]", out["ranks"][0], "preds", p_tail[0, :3].numpy())


def tucker_trunk(m, e, r):
    """TuckER.forward before the x.E^T product (projection.py:322-335), the reference's own tensors."""
    import torch.nn.functional as F
    e1 = F.normalize(m.ent_embeddings(e), p=2, dim=1)
    e1 = m.inp_drop(e1).view(-1, 1, m.d1)
    W_mat = torch.matmul(m.rel_embeddings(r), m.W.weight.view(m.d2, -1)).view(-1, m.d1, m.d1)
    W_mat = m.hidden_dropout1(W_mat)
    x = torch.matmul(e1, W_mat).view(-1, m.d1)
    return m.hidden_dropout2(F.normalize(x, p=2, dim=1))


def make_tucker(name, N, R, d1, d2, b, seed):
    """TuckER (projection.py:258-345): no bias, no reciprocal relations — both directions run the
    same function on (h, r) and (t, r)."""
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1000)
    m = ref_projection.TuckER(tot_entity=N, tot_relation=R, ent_hidden_size=d1, rel_hidden_size=d2, lmbda=0.1,
                              input_dropout=0.0, hidden_dropout1=0.0, hidden_dropout2=0.0)
    with torch.no_grad():
        m.ent_embeddings.weight.normal_(0.0, 0.5)
        m.rel_embeddings.weight.normal_(0.0, 0.5)
        m.W.weight.normal_(0.0, 0.3)
    out = {"N": N, "R": R, "ent_hidden_size": d1, "rel_hidden_size": d2, "label_smoothing": np.float32(LABEL_SMOOTHING)}
    for key, v in m.state_dict().items():
        out["sd_" + key] = v.detach().numpy().copy()
    h = rng.randint(N, size=b).astype(np.int64)
    r = rng.randint(R, size=b).astype(np.int64)
    t = rng.randint(N, size=b).astype(np.int64)
    ht, rt, tt = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)
    out.update(h=h, r=r, t=t)
    m.eval()
    with torch.no_grad():
        x_tail, x_head = tucker_trunk(m, ht, rt), tucker_trunk(m, tt, rt)
        p_tail, p_head = m.forward(ht, rt, direction="tail"), m.forward(tt, rt, direction="head")
        for x, p in ((x_tail, p_tail), (x_head, p_head)):
            assert torch.equal(torch.sigmoid(torch.matmul(x, m.ent_embeddings.weight.T)), p)
    out.update(x_tail=x_tail.numpy().copy(), x_head=x_head.numpy().copy(),
               preds_tail=p_tail.numpy().copy(), preds_head=p_head.numpy().copy())
    q = [(int(h[i]), int(r[i]), int(t[i])) for i in range(N_QUERIES)]
    hr_t, tr_h = mg.random_filters(rng, N, R, q)
    out["ranks"] = mg.reference_ranks(m, N, q, hr_t, tr_h)
    out["filt_t_ptr"], out["filt_t_idx"] = mg.csr(hr_t, [(a, b_) for a, b_, c in q])
    out["filt_h_ptr"], out["filt_h_idx"] = mg.csr(tr_h, [(c, b_) for a, b_, c in q])
    m.train()
    lab_t = (rng.rand(b, N) < 0.03).astype(np.float32)
    lab_h = (rng.rand(b, N) < 0.03).astype(np.float32)
    lab_t[np.arange(b), t] = 1.0
    lab_h[np.arange(b), h] = 1.0
    m.zero_grad()
    loss = Criterion.multi_class_bce(m(tt, rt, direction="head"), m(ht, rt, direction="tail"),
                                     torch.from_numpy(lab_h), torch.from_numpy(lab_t), LABEL_SMOOTHING, N)
    loss.backward()
    out.update(tr_labels_tail=lab_t, tr_labels_head=lab_h, tr_loss=np.float32(loss.item()))
    for key, p in m.named_parameters():
        out["grad_" + key] = p.grad.detach().numpy().copy()
    np.savez_compressed(os.path.join(HERE, name + ".npz"), **out)
    print("wrote", name, "loss", out["tr_loss"], "ranks[0]", out["ranks"][0])


if __name__ == "__main__":
    torch.set_num_threads(1)
    make_tucker("tucker_d32", 97, 5, 32, 16, 24, seed=950)
    for i, (name, N, R, k, k1, b) in enumerate(CASES):
        make_case(name, N, R, k, k1, b, seed=900 + i)
