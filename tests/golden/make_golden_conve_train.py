#!/usr/bin/env python
"""Golden fixtures for ConvE's training-mode trunk kernels by RUNNING THE REFERENCE's class (pykg2vec/models/
projection.py:12-125) in training mode and Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50) on seeded
inputs, torch CPU fp32.

Run where the reference checkout is available (make_golden.py puts it on sys.path):
    python tests/golden/make_golden_conve_train.py

Per case (golden/conve_train/<name>.npz):
  sd_<key>            the reference model's state_dict BEFORE the step (BatchNorm affine parameters and running
                      statistics drawn away from their initial values).  fc.weight ([k, F], 8 MB at k = 200) is
                      np.random.RandomState(fc_seed).standard_normal((k, F)) * fc_scale as fp32, only the seed is stored
  h, r, t             triple ids [b], ids repeating within the batch
  lab_tail / lab_head dense [b, N] labels;  loss = multi_class_bce with label smoothing 0.1
  x_tail / x_head     the trunk's output of each forward (relu(bn2(...)), before the x . E^T product)
  grad_<key>          autograd gradients of `loss` (fc.weight's as a strided sample gradsample_fc.weight)
  sd_after_<key>      the running statistics and num_batches_tracked after both forwards
  noise0/1/2_tail/_head  (dropout case) the noise the reference's inp_drop, feat_drop (Dropout2d: one value per
                      channel) and hidden_drop drew, recovered by replaying each module's draw on a tensor of ones
                      from the saved RNG state and checked against the module's output bit for bit
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402,F401  (installs the import stubs and the reference on sys.path)

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402

OUT_DIR = os.path.join(HERE, "conve_train")
LABEL_SMOOTHING = 0.1
GRAD_SAMPLE_STRIDE = 37
CASES = [
    # name, N, R, k, h1, b, (input_dropout, feature_map_dropout, hidden_dropout), fc.weight from a seed
    ("conve_train_k200_drop", 40, 5, 200, 20, 12, (0.2, 0.2, 0.3), True),
    ("conve_train_12x6", 30, 4, 36, 6, 7, (0.0, 0.0, 0.0), False),
]


def record_dropout(mod, store):
    def pre(m, inp):
        m._rng = torch.get_rng_state()

    def post(m, inp, out):
        after = torch.get_rng_state()
        torch.set_rng_state(m._rng)
        noise = m.forward(torch.ones_like(inp[0]))   # the same module, the same draw (no hooks)
        assert torch.equal(torch.get_rng_state(), after)
        assert torch.equal(out, inp[0] * noise), "dropout is not x * noise"
        store.append(noise.detach().numpy().copy())
    return [mod.register_forward_pre_hook(pre), mod.register_forward_hook(post)]


def make_case(name, N, R, k, h1, b, drops, seeded_fc, seed):
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1000)
    m = ref_projection.ConvE(tot_entity=N, tot_relation=R, hidden_size=k, hidden_size_1=h1, lmbda=0.1,
                             input_dropout=drops[0], feature_map_dropout=drops[1], hidden_dropout=drops[2])
    h2 = k // h1
    F = 32 * (2 * h2 - 2) * (h1 - 2)
    out = {"N": N, "R": R, "hidden_size": k, "hidden_size_1": h1, "drops": np.asarray(drops, dtype=np.float32),
           "label_smoothing": np.float32(LABEL_SMOOTHING)}
    with torch.no_grad():
        for bn in (m.bn0, m.bn1, m.bn2):
            bn.weight.uniform_(0.5, 1.5)
            bn.bias.uniform_(-0.2, 0.2)
            bn.running_mean.uniform_(-0.1, 0.1)
            bn.running_var.uniform_(0.5, 1.5)
        m.b.weight.normal_(0.0, 0.1)
        if seeded_fc:
            out["fc_seed"], out["fc_scale"] = seed + 77, np.float32(0.01)
            w = np.random.RandomState(seed + 77).standard_normal((k, F)) * np.float32(0.01)
            m.fc.weight.copy_(torch.from_numpy(w.astype(np.float32)))
    for key, v in m.state_dict().items():
        if not (seeded_fc and key == "fc.weight"):
            out["sd_" + key] = v.detach().numpy().copy()
    h = rng.randint(N, size=b).astype(np.int64)
    r = rng.randint(R, size=b).astype(np.int64)
    t = rng.randint(N, size=b).astype(np.int64)
    h[1], r[2], t[3] = h[0], r[0], h[0]   # repeated ids: the scatter into the tables accumulates
    ht, rt, tt = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)
    out.update(h=h, r=r, t=t)

    m.train()
    lab_t = (rng.rand(b, N) < 0.05).astype(np.float32)
    lab_h = (rng.rand(b, N) < 0.05).astype(np.float32)
    lab_t[np.arange(b), t] = 1.0
    lab_h[np.arange(b), h] = 1.0
    noises, xs, hooks = [], [], []
    for mod in (m.inp_drop, m.feat_drop, m.hidden_drop):
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
            out["noise0_" + tag] = trio[0].reshape(b, 2 * k)
            out["noise1_" + tag] = trio[1][:, :, 0, 0].copy()
            out["noise2_" + tag] = trio[2].reshape(b, k)
    out.update(lab_tail=lab_t, lab_head=lab_h, loss=np.float32(loss.item()), x_tail=xs[0], x_head=xs[1])
    for key, p in m.named_parameters():
        g = p.grad.detach().numpy().copy()
        if seeded_fc and key == "fc.weight":
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
        make_case(*case, seed=2300 + i)
