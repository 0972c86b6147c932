#!/usr/bin/env python
"""Golden fixtures for AcrE (pykg2vec/models/projection.py:621-746) by RUNNING THE REFERENCE's class and
Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50) on seeded inputs, torch CPU fp32.
Same layout as make_golden_interacte.py's cases (whose helpers this script shares).

Run where the reference checkout is available (make_golden.py puts it on sys.path):
    python tests/golden/make_golden_acre.py

Fixture design.  hidden_size is fixed at 200 by the reference's 10 x 20 view, so fc.weight is [200, C*400] and
the parallel way's W_gate_e.weight is [400, 1600] (2.5 MB in fp32): as random fp32 they and their gradients
would not fit the 1 MB bound on a fixture.  So:
  * after the seeded construction, fc.weight and W_gate_e.weight are REPLACED by small dyadic values,
    n * 2^-8 with n uniform in [-7, 7] (about the scale of their default init), and stored exactly as int8 n
    plus the scale: q_<key> (int8), qscale_<key>;
  * their seeded initial values are kept as a fixed sample of entries plus float64 row sums
    (init_idx_<key>, init_sample_<key>, init_rowsum_<key>), enough to check a seeded construction;
  * their gradients are kept as a fixed sample of entries plus float64 row sums (grad_idx_<key>,
    grad_sample_<key>, grad_rowsum_<key>); every other gradient is stored whole (grad_<key>).

Per case (golden/acre/<name>.npz):
  way (0 serial / 1 parallel), C, atrous [3], acre_bias, N, R, seed
  sd_keys             the reference state_dict's keys in order
  sd_<key>            every other state_dict entry.  ent / rel / conv* / fc.bias / W_gate_e.bias are the seeded
                      initial values (np.random.seed(seed), torch.manual_seed(seed) right before construction);
                      the BN weights and buffers and `bias` are then set to non-trivial values
  h, r, t             triple ids [b]; id 0 occurs in the head, tail and relation columns
  x_tail / x_head     eval-mode trunk output [b,200] — the operand of `x . E^T + bias`, from the reference's own
                      sub-modules (the script asserts sigmoid(x E^T + bias) == model.forward bit for bit)
  preds_tail / _head  eval-mode model.forward(e, r, direction) [b,N]
  ranks               (trank, ftrank, hrank, fhrank) through model.predict_*_rank + MetricCalculator, filtered
  tr_* (train mode, dropouts 0): dense labels, the loss with label smoothing 0.1, autograd gradients (see above)
                      and the BN running statistics after the two forwards (sd_after_<key>)
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
OUT_DIR = os.path.join(HERE, "acre")
CASES = [
    # name, N, R, way, in_channels, (first, second, third) atrous, acre_bias, b
    ("acre_serial_c4", 64, 5, "serial", 4, (1, 3, 5), True, 20),
    ("acre_parallel_c3", 59, 6, "parallel", 3, (2, 11, 23), False, 20),
]
BIG = ("fc.weight", "W_gate_e.weight")
QSCALE = np.float32(2.0 ** -8)
N_SAMPLE = 2048


def trunk(m, e, r):
    """AcrE.forward up to (not including) the x.E^T product, with the reference's own sub-modules
    (projection.py:708-734)."""
    emb_e, emb_r = m.embed2(e, r)
    x = torch.cat([emb_e.view(-1, 1, 10, 20), emb_r.view(-1, 1, 10, 20)], dim=2)
    x = m.bn0(x)
    x = m.inp_drop(x)
    res = x
    if m.way == "serial":
        x = m.conv3(m.conv2(m.conv1(x)))
        x = x + res
    else:
        c1 = m.conv1(x).view(-1, m.in_channels, 400)
        c2 = m.conv2(x).view(-1, m.in_channels, 400)
        c3 = m.conv3(x).view(-1, m.in_channels, 400)
        res = res.expand(-1, m.in_channels, 20, 20).view(-1, m.in_channels, 400)
        x = m.W_gate_e(torch.cat((res, c1, c2, c3), dim=2)).view(-1, m.in_channels, 20, 20)
    x = m.bn1(x)
    x = F.relu(x)
    x = m.feature_map_drop(x)
    x = x.view(x.shape[0], -1)
    x = m.fc(x)
    x = m.hidden_drop(x)
    x = m.bn2(x)
    return F.relu(x)


def sample(rng, a):
    """(flat indices, entries at them, float64 row sums) of a 2-D array"""
    idx = np.sort(rng.choice(a.size, size=min(N_SAMPLE, a.size), replace=False)).astype(np.int64)
    return idx, a.reshape(-1)[idx].copy(), a.astype(np.float64).sum(1)


def make_case(name, N, R, way, C, atrous, acre_bias, b, seed):
    np.random.seed(seed)
    torch.manual_seed(seed)
    m = ref_projection.AcrE(tot_entity=N, tot_relation=R, hidden_size=200, input_dropout=0.0, hidden_dropout=0.0,
                            feature_map_dropout=0.0, in_channels=C, way=way, first_atrous=atrous[0],
                            second_atrous=atrous[1], third_atrous=atrous[2], acre_bias=acre_bias)
    rng = np.random.RandomState(seed + 1000)
    out = {"way": 0 if way == "serial" else 1, "C": C, "atrous": np.array(atrous, dtype=np.int64),
           "acre_bias": int(acre_bias), "N": N, "R": R, "seed": seed,
           "label_smoothing": np.float32(mgp.LABEL_SMOOTHING)}
    sd = m.state_dict()
    out["sd_keys"] = np.array(list(sd))
    with torch.no_grad():
        for key in BIG:
            if key not in sd:
                continue
            out["init_idx_" + key], out["init_sample_" + key], out["init_rowsum_" + key] = \
                sample(rng, sd[key].numpy())
            q = rng.randint(-7, 8, size=tuple(sd[key].shape)).astype(np.int8)
            sd[key].copy_(torch.from_numpy(q.astype(np.float32) * QSCALE))
            out["q_" + key], out["qscale_" + key] = q, QSCALE
        m.bias.normal_(0.0, 0.3)
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.6, 1.4)
            bn.bias.normal_(0.0, 0.2)
            bn.running_mean.normal_(0.0, 0.2)
            bn.running_var.uniform_(0.5, 1.5)
    for key, v in m.state_dict().items():
        if key not in BIG:
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
        g = p.grad.detach().numpy().copy()
        if key in BIG:
            out["grad_idx_" + key], out["grad_sample_" + key], out["grad_rowsum_" + key] = sample(rng, g)
        else:
            out["grad_" + key] = g
    for key, v in mt.state_dict().items():   # BN running statistics after the two training forwards
        if "running" in key:
            out["sd_after_" + key] = v.detach().numpy().copy()
    os.makedirs(OUT_DIR, exist_ok=True)
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    assert os.path.getsize(path) < (1 << 20), "fixture over 1 MB"
    print("wrote", name, os.path.getsize(path), "bytes, loss", out["tr_loss"], "ranks[0]", out["ranks"][0],
          "preds", p_tail[0, :3].numpy())


if __name__ == "__main__":
    torch.set_num_threads(1)
    for i, (name, N, R, way, C, atrous, acre_bias, b) in enumerate(CASES):
        make_case(name, N, R, way, C, atrous, acre_bias, b, seed=1400 + i)
