#!/usr/bin/env python
"""Golden fixtures for AcrE's training-mode trunk kernels by RUNNING THE REFERENCE's class (pykg2vec/models/
projection.py:621-746) in training mode and Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50) on seeded
inputs, torch CPU fp32.

Run where the reference checkout is available (make_golden_proj.py puts it on sys.path):
    python tests/golden/make_golden_acre_train.py

Per case (golden/acre_train/<name>.npz), the layout of make_golden_interacte_train.py:
  way (0 serial / 1 parallel), C, atrous [3], acre_bias, N, R   the configuration
  sd_<key>            the reference model's state_dict BEFORE the step (BatchNorm affine parameters and running
                      statistics drawn away from their initial values).  The large weights named in `seeded`
                      (fc.weight [200, C*400]; W_gate_e.weight [400, 1600]) are
                      np.random.RandomState(seed_<key>).standard_normal(shape) * scale_<key> as fp32; only the seed
                      and scale are stored
  h, r, t             triple ids [b]: ids repeat within the batch in every column, and one entity is both a head and
                      a tail
  lab_tail / lab_head dense [b, N] labels;  loss = multi_class_bce with label smoothing 0.1
  x_tail / x_head     the trunk's output of each forward (relu(bn2(...)), before the x . E^T product)
  grad_<key>          autograd gradients of `loss` (a seeded weight's as a strided sample gradsample_<key>)
  sd_after_<key>      the running statistics and num_batches_tracked after both forwards
  noise0/1/2_tail/_head  (dropout case) the noise the reference's inp_drop ([b, 400]), feature_map_drop (Dropout2d:
                      [b, C]) and hidden_drop ([b, 200]) drew, recovered as make_golden_conve_train.record_dropout does
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden_proj  # noqa: E402,F401  (installs the import stubs and the reference on sys.path)
from make_golden_conve_train import GRAD_SAMPLE_STRIDE, LABEL_SMOOTHING, record_dropout  # noqa: E402

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402

OUT_DIR = os.path.join(HERE, "acre_train")
CASES = [
    # name, N, R, way, C, atrous, acre_bias, b, (input, feature_map, hidden dropout), seeded weights
    ("acre_train_serial_c32_drop", 40, 6, "serial", 32, (1, 2, 2), True, 6, (0.3, 0.2, 0.5), ("fc.weight",)),
    ("acre_train_parallel_c3", 30, 5, "parallel", 3, (2, 11, 23), False, 5, (0.0, 0.0, 0.0),
     ("fc.weight", "W_gate_e.weight")),
]
SEEDED_SCALE = {"fc.weight": 0.005, "W_gate_e.weight": 0.02}


def seeded_weight(seed, scale, shape):
    return (np.random.RandomState(seed).standard_normal(shape) * np.float32(scale)).astype(np.float32)


def make_case(name, N, R, way, C, atrous, bias, b, drops, seeded, seed):
    np.random.seed(seed)
    torch.manual_seed(seed)
    m = ref_projection.AcrE(tot_entity=N, tot_relation=R, hidden_size=200, input_dropout=drops[0],
                            hidden_dropout=drops[2], feature_map_dropout=drops[1], in_channels=C, way=way,
                            first_atrous=atrous[0], second_atrous=atrous[1], third_atrous=atrous[2], acre_bias=bias)
    rng = np.random.RandomState(seed + 1000)
    out = {"N": N, "R": R, "way": 0 if way == "serial" else 1, "C": C, "atrous": np.asarray(atrous, np.int64),
           "acre_bias": bool(bias), "drops": np.asarray(drops, dtype=np.float32),
           "label_smoothing": np.float32(LABEL_SMOOTHING), "seeded": np.asarray(seeded)}
    params = dict(m.named_parameters())
    with torch.no_grad():
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
        m.bias.normal_(0.0, 0.1)
        for i, key in enumerate(seeded):
            out["seed_" + key], out["scale_" + key] = seed + 77 + i, np.float32(SEEDED_SCALE[key])
            w = seeded_weight(seed + 77 + i, SEEDED_SCALE[key], tuple(params[key].shape))
            params[key].copy_(torch.from_numpy(w))
    for key, v in m.state_dict().items():
        if key not in seeded:
            out["sd_" + key] = v.detach().numpy().copy()
    h = rng.randint(0, N, size=b).astype(np.int64)
    r = rng.randint(0, R, size=b).astype(np.int64)
    t = rng.randint(0, N, size=b).astype(np.int64)
    h[2], r[3], t[4] = h[0], r[0], t[1]            # repeated ids in every column: the scatter must accumulate
    r[1] = r[0]
    t[3] = h[0]                                    # an entity both a head (tail direction) and a tail (head direction)
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
            out["noise0_" + tag] = trio[0].reshape(b, 400)
            out["noise1_" + tag] = trio[1][:, :, 0, 0].copy()
            out["noise2_" + tag] = trio[2].reshape(b, 200)
    out.update(lab_tail=lab_t, lab_head=lab_h, loss=np.float32(loss.item()), x_tail=xs[0], x_head=xs[1])
    for key, p in m.named_parameters():
        g = p.grad.detach().numpy().copy()
        if key in seeded:
            out["gradsample_" + key] = g.reshape(-1)[::GRAD_SAMPLE_STRIDE].copy()
        else:
            out["grad_" + key] = g
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
        make_case(*case, seed=2900 + i)
