#!/usr/bin/env python
"""Golden fixtures for HypER's training-mode trunk kernels by RUNNING THE REFERENCE's class (pykg2vec/models/
projection.py:508-618) in training mode and Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50) on seeded
inputs, torch CPU fp32.

Run where the reference checkout is available (make_golden.py puts it on sys.path):
    python tests/golden/make_golden_hyper_train.py

Per case (golden/hyper_train/<name>.npz), the layout of make_golden_conve_train.py:
  sd_<key>            the reference model's state_dict BEFORE the step (BatchNorm affine parameters and running
                      statistics drawn away from their initial values).  fc.weight ([de, F], 4.9 MB at de = 200) is
                      np.random.RandomState(fc_seed).standard_normal((de, F)) * fc_scale as fp32, only the seed is stored
  h, r, t             triple ids [b]: ids repeat within the batch, and id 0 (padding_idx of both embeddings) occurs in
                      the head, tail and relation columns
  lab_tail / lab_head dense [b, N] labels;  loss = multi_class_bce with label smoothing 0.1
  x_tail / x_head     the trunk's output of each forward (relu(bn2(...)), before the x . E^T product)
  grad_<key>          autograd gradients of `loss` (fc.weight's as a strided sample gradsample_fc.weight)
  sd_after_<key>      the running statistics and num_batches_tracked after both forwards
  noise0/1/2_tail/_head  (dropout case) the noise the reference's inp_drop, feature_map_drop (Dropout2d: one value
                      per channel) and hidden_drop drew, recovered as make_golden_conve_train.record_dropout does
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_conve_train import GRAD_SAMPLE_STRIDE, LABEL_SMOOTHING, record_dropout  # noqa: E402

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402

OUT_DIR = os.path.join(HERE, "hyper_train")
CASES = [
    # name, N, R, de, dr, b, (input_dropout, feature_map_dropout, hidden_dropout), fc.weight from a seed
    ("hyper_train_d200_drop", 40, 6, 200, 200, 12, (0.3, 0.2, 0.3), True),
    ("hyper_train_24x10", 30, 5, 24, 10, 7, (0.0, 0.0, 0.0), False),
]


def make_case(name, N, R, de, dr, b, drops, seeded_fc, seed):
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1000)
    m = ref_projection.HypER(tot_entity=N, tot_relation=R, ent_hidden_size=de, rel_hidden_size=dr,
                             input_dropout=drops[0], feature_map_dropout=drops[1], hidden_dropout=drops[2],
                             device="cpu")
    F = 32 * (de - 8)
    out = {"N": N, "R": R, "ent_hidden_size": de, "rel_hidden_size": dr, "drops": np.asarray(drops, dtype=np.float32),
           "label_smoothing": np.float32(LABEL_SMOOTHING)}
    with torch.no_grad():
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
        m.b.normal_(0.0, 0.1)
        if seeded_fc:
            out["fc_seed"], out["fc_scale"] = seed + 77, np.float32(0.01)
            w = np.random.RandomState(seed + 77).standard_normal((de, F)) * np.float32(0.01)
            m.fc.weight.copy_(torch.from_numpy(w.astype(np.float32)))
    for key, v in m.state_dict().items():
        if not (seeded_fc and key == "fc.weight"):
            out["sd_" + key] = v.detach().numpy().copy()
    h = rng.randint(1, N, size=b).astype(np.int64)
    r = rng.randint(1, R, size=b).astype(np.int64)
    t = rng.randint(1, N, size=b).astype(np.int64)
    h[0], t[1], r[0], r[3] = 0, 0, 0, 0            # the padding rows take part (forward and gradients)
    h[2], r[4], t[3] = h[1], r[1], h[1]            # repeated ids: the scatter into the tables accumulates
    ht, rt, tt = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)
    out.update(h=h, r=r, t=t)

    m.train()
    lab_t = (rng.rand(b, N) < 0.05).astype(np.float32)
    lab_h = (rng.rand(b, N) < 0.05).astype(np.float32)
    lab_t[np.arange(b), t] = 1.0
    lab_h[np.arange(b), h] = 1.0
    noises, xs, hooks = [], [], []
    for mod in (m.inp_drop, m.feature_map_drop, m.hidden_drop):
        hooks += record_dropout(mod, noises)
    hooks.append(m.bn2.register_forward_hook(lambda mod, inp, o: xs.append(torch.relu(o).detach().numpy().copy())))
    m.zero_grad()
    pred_tails = m(ht, rt, direction="tail")
    pred_heads = m(tt, rt, direction="head")
    for hk in hooks:
        hk.remove()
    loss = Criterion.multi_class_bce(pred_heads, pred_tails, torch.from_numpy(lab_h), torch.from_numpy(lab_t),
                                     LABEL_SMOOTHING, N)
    loss.backward()
    assert len(noises) == 6 and len(xs) == 2
    if any(drops):
        for tag, trio in (("tail", noises[:3]), ("head", noises[3:])):
            out["noise0_" + tag] = trio[0].reshape(b, de)
            out["noise1_" + tag] = trio[1][:, :, 0, 0].copy()
            out["noise2_" + tag] = trio[2].reshape(b, de)
    out.update(lab_tail=lab_t, lab_head=lab_h, loss=np.float32(loss.item()), x_tail=xs[0], x_head=xs[1])
    for key, p in m.named_parameters():
        g = p.grad.detach().numpy().copy()
        if seeded_fc and key == "fc.weight":
            out["gradsample_" + key] = g.reshape(-1)[::GRAD_SAMPLE_STRIDE].copy()
        else:
            out["grad_" + key] = g
    assert not out["grad_rel_embeddings.weight"][0].any() and out["grad_ent_embeddings.weight"][0].any()
    for key, v in m.state_dict().items():
        if "running" in key or "num_batches" in key:
            out["sd_after_" + key] = v.detach().numpy().copy()
    os.makedirs(OUT_DIR, exist_ok=True)
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    assert os.path.getsize(path) < (1 << 20), "fixture over 1 MB"
    print("wrote", name, os.path.getsize(path), "bytes, loss", out["loss"])


if __name__ == "__main__":
    torch.set_num_threads(1)
    for i, case in enumerate(CASES):
        make_case(*case, seed=2600 + i)
