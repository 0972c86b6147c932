#!/usr/bin/env python
"""Golden fixtures for TuckER's trunk kernels by RUNNING THE REFERENCE's class (pykg2vec/models/projection.py:258-345)
and Criterion.multi_class_bce (pykg2vec/utils/criterion.py:41-50) on seeded inputs, torch CPU fp32.

Run where the reference checkout is available (make_golden.py puts it on sys.path):
    python tests/golden/make_golden_tucker.py

Per case (golden/tucker/<name>.npz):
  sd_<key>            the reference model's state_dict.  The d1 = d2 = 200 case would need 32 MB for W: there W is
                      np.random.RandomState(W_seed).standard_normal((d2, d1*d1)) * W_scale as fp32 (a stable numpy
                      stream), and only W_seed / W_scale are stored
  h, r, t             triple ids [b]: some relations repeat within the batch, others never occur
  preds_tail / _head  eval-mode model.forward(e, r, direction) [b, N]
  ranks               (trank, ftrank, hrank, fhrank) of the first n_queries triples through the reference Evaluator
                      walk; only queries whose target prediction is at least MIN_GAP away from every other entity's
                      are kept (n_ambiguous counts the ones dropped), so the ranks do not hinge on rounding
  lab_tail / lab_head dense [b, N] labels;  loss = multi_class_bce with label smoothing 0.1, training mode
  grad_<key>          autograd gradients of `loss` (W's as a strided sample gradsample_W.weight for the large case)
  noise0/1/2_tail/_head  (dropout case) the noise the reference's three nn.Dropout modules drew in each forward,
                      recovered by replaying the module's draw on a tensor of ones from the saved RNG state and
                      checked against the module's output bit for bit
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402  (installs the import stubs and the reference on sys.path)

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402

OUT_DIR = os.path.join(HERE, "tucker")
LABEL_SMOOTHING = 0.1
MIN_GAP = 1e-5
GRAD_SAMPLE_STRIDE = 61
CASES = [
    # name, N, R, d1, d2, b, (input_dropout, hidden_dropout1, hidden_dropout2), W from a seed
    ("tucker_d200", 61, 12, 200, 200, 16, (0.0, 0.0, 0.0), True),
    ("tucker_33x7", 83, 9, 33, 7, 14, (0.0, 0.0, 0.0), False),
    ("tucker_50x30_drop", 71, 8, 50, 30, 10, (0.3, 0.4, 0.5), False),
]


def record_dropout(mod, store):
    def pre(m, inp):
        m._rng = torch.get_rng_state()

    def post(m, inp, out):
        after = torch.get_rng_state()
        torch.set_rng_state(m._rng)
        noise = torch.nn.functional.dropout(torch.ones_like(inp[0]), m.p, m.training)
        assert torch.equal(torch.get_rng_state(), after)
        assert torch.equal(out, inp[0] * noise), "nn.Dropout is not x * noise"
        store.append(noise.detach().numpy().copy())
    return [mod.register_forward_pre_hook(pre), mod.register_forward_hook(post)]


def make_case(name, N, R, d1, d2, b, drops, seeded_W, seed):
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1000)
    m = ref_projection.TuckER(tot_entity=N, tot_relation=R, ent_hidden_size=d1, rel_hidden_size=d2, lmbda=0.1,
                              input_dropout=drops[0], hidden_dropout1=drops[1], hidden_dropout2=drops[2])
    out = {"N": N, "R": R, "d1": d1, "d2": d2, "drops": np.asarray(drops, dtype=np.float32),
           "label_smoothing": np.float32(LABEL_SMOOTHING)}
    with torch.no_grad():
        m.ent_embeddings.weight.normal_(0.0, 0.5)
        m.rel_embeddings.weight.normal_(0.0, 0.5)
        if seeded_W:
            out["W_seed"], out["W_scale"] = seed + 77, np.float32(0.3)
            w = np.random.RandomState(seed + 77).standard_normal((d2, d1 * d1)) * np.float32(0.3)
            m.W.weight.copy_(torch.from_numpy(w.astype(np.float32)))
        else:
            m.W.weight.normal_(0.0, 0.3)
    for key, v in m.state_dict().items():
        if not (seeded_W and key == "W.weight"):
            out["sd_" + key] = v.detach().numpy().copy()
    present = rng.choice(R, size=max(2, R // 2), replace=False)   # half of the relations never occur
    h = rng.randint(N, size=b).astype(np.int64)
    r = present[rng.randint(len(present), size=b)].astype(np.int64)
    t = rng.randint(N, size=b).astype(np.int64)
    ht, rt, tt = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)
    out.update(h=h, r=r, t=t)

    m.eval()
    with torch.no_grad():
        p_tail, p_head = m.forward(ht, rt, direction="tail"), m.forward(tt, rt, direction="head")
    out.update(preds_tail=p_tail.numpy().copy(), preds_head=p_head.numpy().copy())
    keep = []
    for i in range(b):
        gaps = []
        for p, tgt in ((p_tail[i], t[i]), (p_head[i], h[i])):
            d = (p - p[tgt]).abs()
            d[tgt] = 1.0
            gaps.append(float(d.min()))
        if min(gaps) >= MIN_GAP:
            keep.append(i)
    out["n_ambiguous"] = b - len(keep)
    out["query_rows"] = np.asarray(keep, dtype=np.int64)
    q = [(int(h[i]), int(r[i]), int(t[i])) for i in keep]
    hr_t, tr_h = mg.random_filters(rng, N, R, q, extra=20)
    out["ranks"] = mg.reference_ranks(m, N, q, hr_t, tr_h)
    out["filt_t_ptr"], out["filt_t_idx"] = mg.csr(hr_t, [(a, b_) for a, b_, c in q])
    out["filt_h_ptr"], out["filt_h_idx"] = mg.csr(tr_h, [(c, b_) for a, b_, c in q])

    m.train()
    lab_t = (rng.rand(b, N) < 0.05).astype(np.float32)
    lab_h = (rng.rand(b, N) < 0.05).astype(np.float32)
    lab_t[np.arange(b), t] = 1.0
    lab_h[np.arange(b), h] = 1.0
    noises, hooks = [], []
    for mod in (m.inp_drop, m.hidden_dropout1, m.hidden_dropout2):
        hooks += record_dropout(mod, noises)
    m.zero_grad()
    pred_tails = m(ht, rt, direction="tail")
    pred_heads = m(tt, rt, direction="head")
    for hk in hooks:
        hk.remove()
    loss = Criterion.multi_class_bce(pred_heads, pred_tails, torch.from_numpy(lab_h), torch.from_numpy(lab_t),
                                     LABEL_SMOOTHING, N)
    loss.backward()
    assert len(noises) == 6
    if any(drops):
        for tag, trio in (("tail", noises[:3]), ("head", noises[3:])):
            out["noise0_" + tag] = trio[0].reshape(b, d1)
            out["noise1_" + tag] = trio[1].reshape(b, d1, d1)
            out["noise2_" + tag] = trio[2].reshape(b, d1)
    out.update(lab_tail=lab_t, lab_head=lab_h, loss=np.float32(loss.item()),
               tr_preds_tail=pred_tails.detach().numpy().copy(), tr_preds_head=pred_heads.detach().numpy().copy())
    for key, p in m.named_parameters():
        g = p.grad.detach().numpy().copy()
        if seeded_W and key == "W.weight":
            out["gradsample_" + key] = g.reshape(-1)[::GRAD_SAMPLE_STRIDE].copy()
        else:
            out["grad_" + key] = g
    os.makedirs(OUT_DIR, exist_ok=True)
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    assert os.path.getsize(path) < (1 << 20), "fixture over 1 MB"
    print("wrote", name, os.path.getsize(path), "bytes, loss", out["loss"], "queries", len(keep), "ambiguous",
          out["n_ambiguous"], "distinct relations", len(np.unique(r)), "of", R)


if __name__ == "__main__":
    torch.set_num_threads(1)
    for i, case in enumerate(CASES):
        make_case(*case, seed=1700 + i)
