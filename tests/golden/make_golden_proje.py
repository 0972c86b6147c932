#!/usr/bin/env python
"""Golden fixtures for ProjE_pointwise (pykg2vec/models/projection.py:128-257) by RUNNING THE REFERENCE's class,
Criterion.multi_class (pykg2vec/utils/criterion.py:52-55) and get_reg on seeded inputs, torch CPU fp32.
torch.dropout is wrapped only to record the noise the reference drew: the wrapper draws it once more from the
same RNG state on a tensor of ones, restores the state, calls the real torch.dropout and checks that its output
is x * noise bit for bit.

Run where the reference checkout is available (make_golden.py puts it on sys.path):
    python tests/golden/make_golden_proje.py

Per case (golden/proje/<name>.npz):
  sd_<key>            the reference model's state_dict (the eight tables)
  h, r, t             triple ids [b]
  lab_tail / lab_head dense [b, N] labels as process_function_multiclass builds them with neg_rate > 0
                      (generator.py:200-238): 1 at the positives, -1 at the first min(100, N) ids of one
                      permutation unless positive, 0 elsewhere; the same negatives in every row and direction
  noise_tail / _head  the dropout noise the reference drew in forward() (ones when hidden_dropout = 0)
  x_tail / x_head     f1(h, r) / f2(t, r) without dropout [b, k] (the evaluation trunk)
  loss_tail / _head   forward(e, r, labels, direction);  reg = get_reg;  loss = multi_class(heads, tails) + reg
  grad_<key>          autograd gradient of `loss` for every parameter
  ranks               (trank, ftrank, hrank, fhrank) through predict_*_rank + MetricCalculator, filtered
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

OUT_DIR = os.path.join(HERE, "proje")
N_QUERIES = 6
CASES = [
    # name, N, R, k, b, hidden_dropout, lmbda, heavy rows
    ("proje_n60", 60, 5, 16, 12, 0.5, 1e-3, 0),      # N < 100: every non-positive entity is a negative
    ("proje_n300", 300, 7, 24, 16, 0.5, 1e-3, 0),
    ("proje_heavy", 150, 4, 16, 10, 0.0, 1e-3, 12),  # saturated sigmoids: both clamps clip, sigmoid ties at 1
]


def recording_dropout(store):
    real = torch.dropout

    def dropout(x, p, train):
        state = torch.get_rng_state()
        noise = real(torch.ones_like(x), p, train)
        torch.set_rng_state(state)
        out = real(x, p, train)
        assert torch.equal(out, x * noise), "torch.dropout is not x * noise"
        store.append(noise.detach().clone())
        return out
    return dropout


def make_case(name, N, R, k, b, p, lmbda, heavy, seed):
    torch.manual_seed(seed)
    rng = np.random.RandomState(seed + 1000)
    m = ref_projection.ProjE_pointwise(tot_entity=N, tot_relation=R, hidden_size=k, lmbda=lmbda, hidden_dropout=p,
                                       device="cpu")
    heavy_ids = np.zeros(0, dtype=np.int64)
    if heavy:
        with torch.no_grad():
            for emb in (m.De1, m.Dr1, m.De2, m.Dr2):
                emb.weight.uniform_(-3.0, 3.0)
            m.bc1.weight.uniform_(-1.0, 1.0)
            m.bc2.weight.uniform_(-1.0, 1.0)
            heavy_ids = rng.choice(N, heavy, replace=False).astype(np.int64)
            m.ent_embeddings.weight[torch.from_numpy(heavy_ids)] *= 200.0
    out = {"N": N, "R": R, "k": k, "hidden_dropout": np.float32(p), "lmbda": np.float32(lmbda), "heavy": heavy_ids}
    for key, v in m.state_dict().items():
        out["sd_" + key] = v.detach().numpy().copy()
    light = np.setdiff1d(np.arange(N), heavy_ids)
    h = rng.choice(light, size=b).astype(np.int64)
    r = rng.randint(R, size=b).astype(np.int64)
    t = rng.choice(light, size=b).astype(np.int64)
    triples = [(int(h[i]), int(r[i]), int(t[i])) for i in range(b)]
    hr_t, tr_h = mg.random_filters(rng, N, R, triples, extra=6)
    for i in range(0, b, 3):                # heavy entities among the positives too
        if heavy:
            hr_t[(int(h[i]), int(r[i]))].add(int(heavy_ids[i % heavy]))
            tr_h[(int(t[i]), int(r[i]))].add(int(heavy_ids[(i + 1) % heavy]))
    random_ids = rng.permutation(N)
    lab_t = np.zeros((b, N), dtype=np.float32)
    lab_h = np.zeros((b, N), dtype=np.float32)
    for i, (hh, rr, tt) in enumerate(triples):
        for lab, pos in ((lab_t, hr_t[(hh, rr)]), (lab_h, tr_h[(tt, rr)])):
            lab[i, sorted(pos)] = 1.0
            for idx in random_ids[0:100]:
                if idx not in pos:
                    lab[i, idx] = -1.0
    out.update(h=h, r=r, t=t, lab_tail=lab_t, lab_head=lab_h)
    ht, rt, tt_ = torch.from_numpy(h), torch.from_numpy(r), torch.from_numpy(t)

    # ---- training: trainer.py:167-172 (train_step_projection, ProjE branch) + loss.backward() ---------------
    noises = []
    real = torch.dropout
    torch.dropout = recording_dropout(noises)
    try:
        m.zero_grad()
        pred_tails = m(ht, rt, torch.from_numpy(lab_t), direction="tail")
        pred_heads = m(tt_, rt, torch.from_numpy(lab_h), direction="head")
    finally:
        torch.dropout = real
    reg = m.get_reg(ht, rt, tt_)
    loss = Criterion.multi_class(pred_heads, pred_tails) + reg
    loss.backward()
    assert len(noises) == 2
    out.update(noise_tail=noises[0].numpy().copy(), noise_head=noises[1].numpy().copy(),
               loss_tail=np.float32(pred_tails.item()), loss_head=np.float32(pred_heads.item()),
               reg=np.float32(reg.item()), loss=np.float32(loss.item()))
    for key, prm in m.named_parameters():
        out["grad_" + key] = prm.grad.detach().numpy().copy()

    # ---- evaluation trunk and ranks --------------------------------------------------------------------------
    with torch.no_grad():
        E, Rl = m.ent_embeddings.weight, m.rel_embeddings.weight
        out["x_tail"] = m.f1(E[ht], Rl[rt]).numpy().copy()
        out["x_head"] = m.f2(E[tt_], Rl[rt]).numpy().copy()
    q = triples[:N_QUERIES]
    fhr_t, ftr_h = mg.random_filters(rng, N, R, q)
    out["ranks"] = mg.reference_ranks(m, N, q, fhr_t, ftr_h)
    out["filt_t_ptr"], out["filt_t_idx"] = mg.csr(fhr_t, [(a, b_) for a, b_, c in q])
    out["filt_h_ptr"], out["filt_h_idx"] = mg.csr(ftr_h, [(c, b_) for a, b_, c in q])
    os.makedirs(OUT_DIR, exist_ok=True)
    path = os.path.join(OUT_DIR, name + ".npz")
    np.savez_compressed(path, **out)
    assert os.path.getsize(path) < (1 << 20), "fixture over 1 MB"
    print("wrote", name, "loss", out["loss"], "reg", out["reg"], "ranks[0]", out["ranks"][0],
          "labels +%d -%d" % ((lab_t > 0).sum(), (lab_t < 0).sum()))


if __name__ == "__main__":
    torch.set_num_threads(1)
    for i, case in enumerate(CASES):
        make_case(*case, seed=1500 + i)
