#!/usr/bin/env python
"""Golden fixtures for InteractE (pykg2vec/models/projection.py:347-505) by RUNNING THE REFERENCE's class
and Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50) on seeded inputs, torch CPU fp32.
Same layout as make_golden_hyper.py's cases (whose helpers this script shares).

Run where the reference checkout is available (make_golden.py puts it on sys.path):
    python tests/golden/make_golden_interacte.py

Per case (golden/interacte/<name>.npz):
  P, F, ks, reshape_height, reshape_width, N, R, seed
  chequer_perm        the model's chequer permutation [P, 2k] (not in state_dict): np.random.seed(seed) and
                      torch.manual_seed(seed) right before construction
  sd_<key>            the reference model's full state_dict.  ent / rel / conv_filt / fc are the seeded initial
                      values; the BN weights and buffers and `bias` are then set to non-trivial values
  h, r, t             triple ids [b]; id 0 occurs in the head, tail and relation columns
  x_tail / x_head     eval-mode trunk output [b,k] — the operand of `x . E^T + bias`, from the reference's own
                      sub-modules (the script asserts sigmoid(x E^T + bias) == model.forward bit for bit)
  preds_tail / _head  eval-mode model.forward(e, r, direction) [b,N]
  ranks               (trank, ftrank, hrank, fhrank) through model.predict_*_rank + MetricCalculator, filtered
  tr_* (train mode, dropouts 0): dense labels, the loss with label smoothing 0.1, autograd gradients of every
                      parameter (grad_<key>) and the BN running statistics after the two forwards
"""
import copy
import os
import sys

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_proj as mgp  # noqa: E402  (installs the import stubs and the reference on sys.path)

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402

mg = mgp.mg
OUT_DIR = os.path.join(HERE, "interacte")
CASES = [
    # name, N, R, P, F, ks, reshape_height, reshape_width, b   (image: 2*reshape_width rows x reshape_height cols)
    ("interacte_p2", 97, 5, 2, 6, 5, 6, 4, 24),
    ("interacte_p3", 113, 6, 3, 4, 7, 8, 5, 20),
]


def trunk(m, e, r):
    """InteractE.forward up to (not including) the x.E^T product, with the reference's own sub-modules
    (projection.py:427-442)."""
    emb_e, emb_r = m.embed2(e, r)
    comb = torch.cat([emb_e, emb_r], dim=-1)
    x = comb[:, m.chequer_perm].reshape((-1, m.feature_permutation, 2 * m.reshape_width, m.reshape_height))
    x = m.bn0(x)
    x = m.inp_drop(x)
    x = ref_projection.InteractE._circular_padding_chw(x, m.kernel_size // 2)
    x = F.conv2d(x, m.conv_filt.repeat(m.feature_permutation, 1, 1, 1), padding=m.padding,
                 groups=m.feature_permutation)
    x = m.bn1(x)
    x = F.relu(x)
    x = m.feature_map_drop(x)
    x = x.view(-1, m.flat_sz)
    x = m.fc(x)
    x = m.hidden_drop(x)
    x = m.bn2(x)
    return F.relu(x)


def make_case(name, N, R, P, Fn, ks, rh, rw, b, seed):
    np.random.seed(seed)
    torch.manual_seed(seed)
    m = ref_projection.InteractE(tot_entity=N, tot_relation=R, hidden_size=rh * rw, input_dropout=0.0,
                                 hidden_dropout=0.0, feature_map_dropout=0.0, feature_permutation=P,
                                 num_filters=Fn, kernel_size=ks, reshape_height=rh, reshape_width=rw, device="cpu")
    rng = np.random.RandomState(seed + 1000)
    with torch.no_grad():
        m.bias.normal_(0.0, 0.3)
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.6, 1.4)
            bn.bias.normal_(0.0, 0.2)
            bn.running_mean.normal_(0.0, 0.2)
            bn.running_var.uniform_(0.5, 1.5)
    out = {"N": N, "R": R, "P": P, "F": Fn, "ks": ks, "reshape_height": rh, "reshape_width": rw, "seed": seed,
           "label_smoothing": np.float32(mgp.LABEL_SMOOTHING),
           "chequer_perm": m.chequer_perm.numpy().astype(np.int64)}
    for key, v in m.state_dict().items():
        out["sd_" + key] = v.detach().numpy().copy()
    h = rng.randint(N, size=b).astype(np.int64)
    r = rng.randint(R, size=b).astype(np.int64)
    t = rng.randint(N, size=b).astype(np.int64)
    h[0], t[1], r[0], r[2] = 0, 0, 0, 0
    ht, rt, tt = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)
    out.update(h=h, r=r, t=t)

    # ---- eval mode ---------------------------------------------------------------------------
    m.eval()
    with torch.no_grad():
        x_tail, x_head = trunk(m, ht, rt), trunk(m, tt, rt)
        p_tail = m.forward(ht, rt, direction="tail")
        p_head = m.forward(tt, rt, direction="head")
        for x, p in ((x_tail, p_tail), (x_head, p_head)):
            again = torch.mm(x, m.ent_embeddings.weight.transpose(1, 0))
            again += m.bias.expand_as(again)
            assert torch.equal(torch.sigmoid(again), p), "trunk() is not what the reference forward evaluates"
    assert (x_tail > 0).any() and (x_tail == 0).any()
    out.update(x_tail=x_tail.numpy().copy(), x_head=x_head.numpy().copy(),
               preds_tail=p_tail.numpy().copy(), preds_head=p_head.numpy().copy())
    q = [(int(h[i]), int(r[i]), int(t[i])) for i in range(mgp.N_QUERIES)]
    hr_t, tr_h = mg.random_filters(rng, N, R, q)
    out["ranks"] = mg.reference_ranks(m, N, q, hr_t, tr_h)
    out["filt_t_ptr"], out["filt_t_idx"] = mg.csr(hr_t, [(a, b_) for a, b_, c in q])
    out["filt_h_ptr"], out["filt_h_idx"] = mg.csr(tr_h, [(c, b_) for a, b_, c in q])

    # ---- train mode: trainer.py:159-166 (train_step_projection) + criterion.py:41-50 -----------
    mt = copy.deepcopy(m)
    mt.train()
    lab_t = (rng.rand(b, N) < 0.03).astype(np.float32)
    lab_h = (rng.rand(b, N) < 0.03).astype(np.float32)
    lab_t[np.arange(b), t] = 1.0
    lab_h[np.arange(b), h] = 1.0
    mt.zero_grad()
    pred_tails = mt(ht, rt, direction="tail")
    pred_heads = mt(tt, rt, direction="head")
    loss = Criterion.multi_class_bce(pred_heads, pred_tails, torch.from_numpy(lab_h), torch.from_numpy(lab_t),
                                     mgp.LABEL_SMOOTHING, N)
    loss.backward()
    out.update(tr_labels_tail=lab_t, tr_labels_head=lab_h, tr_loss=np.float32(loss.item()),
               tr_preds_tail=pred_tails.detach().numpy().copy(), tr_preds_head=pred_heads.detach().numpy().copy())
    for key, p in mt.named_parameters():
        out["grad_" + key] = p.grad.detach().numpy().copy()
    for key, v in mt.state_dict().items():   # BN running statistics after the two training forwards
        if "running" in key:
            out["sd_after_" + key] = v.detach().numpy().copy()
    os.makedirs(OUT_DIR, exist_ok=True)
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    assert os.path.getsize(path) < (1 << 20), "fixture over 1 MB"
    print("wrote", name, "loss", out["tr_loss"], "ranks[0]", out["ranks"][0], "preds", p_tail[0, :3].numpy())


if __name__ == "__main__":
    torch.set_num_threads(1)
    for i, (name, N, R, P, Fn, ks, rh, rw, b) in enumerate(CASES):
        make_case(name, N, R, P, Fn, ks, rh, rw, b, seed=1300 + i)
