#!/usr/bin/env python
"""ProjE_pointwise timings (NOT bench.py, which times the flagship workload) on the FB15k-237 shape (N = 14,541,
R = 237, k = 200, B = 200; hyperparams/ProjE_pointwise.yaml: adam, lr 0.01, hidden_dropout 0.5, lmbda 1e-5), CUDA
events, L2 flushed before every repetition.  One JSON line per measurement, each carrying the card's name and power
limit read in the same run (nvidia-smi --query-gpu, read only):

  train step   the fused step on device labels: kge_proje_train_step (both directions, labelled entries only)
               + kge_reg_l1_dense + kge_optim_apply_dense over the eight tables, against the reference's dense
               formulation in torch ops on the same card: tanh trunk + dropout, sigmoid(x E^T) over all N,
               the clamped log loss over the dense [B, N] labels, get_reg, autograd backward and torch.optim.Adam
  rank e2e     Evaluator.rank_triples for 512 filtered queries (host ids in, ranks out): trunk + kge_proj_rank

Label rows: each row holds 1 to 30 positives and the batch's 100 shared negatives, as the Generator builds them
with neg_rate > 0.  Inputs are fixed-seed.

    python bench_proje.py [--reps 20] [--out results/proje.jsonl]
"""
import argparse
import json
import os
import subprocess
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from pykg2vec_b200 import _lib, import_model  # noqa: E402

N, R, K, B, Q = 14541, 237, 200, 200, 512
LR, DROPOUT, LMBDA = 0.01, 0.5, 1e-5


def card():
    """(name, power limit) of GPU 0 as nvidia-smi reports them: the limit in W, or nvidia-smi's own text"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,enforced.power.limit",
                              "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as exc:
        return "unknown (%s)" % exc, None
    fields = [f.strip() for f in out.split(",")]
    for v in fields[1:]:
        try:
            return fields[0], float(v)
        except ValueError:
            pass
    return fields[0], " / ".join(fields[1:]) or None


def time_ms(fn, reps, flush):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    total = 0.0
    for _ in range(reps):
        flush.zero_()                    # 256 MiB > the 50 MB L2
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        total += a.elapsed_time(b)
    return total / reps


def dense_reference_step(m, opt, h, r, t, hr_t, tr_h):
    """projection.py:194-210 (+ get_reg :189-192) in torch ops over all N entities, autograd, torch Adam"""
    opt.zero_grad()
    E, Rl = m.ent_embeddings.weight, m.rel_embeddings.weight
    zero = torch.zeros(1, device=E.device)
    total = 0
    for e, lab, De, Dr, bc in ((h, hr_t, m.De1, m.Dr1, m.bc1), (t, tr_h, m.De2, m.Dr2, m.bc2)):
        x = torch.tanh(E[e] * De.weight + Rl[r] * Dr.weight + bc.weight)
        s = torch.sigmoid(torch.matmul(torch.dropout(x, p=DROPOUT, train=True), E.T))
        total = total - torch.sum(torch.log(torch.clamp(s, 1e-10, 1.0)) * torch.max(zero, lab)) \
            - torch.sum(torch.log(torch.clamp(1 - s, 1e-10, 1.0)) * torch.max(zero, torch.neg(lab)))
    reg = LMBDA * (torch.sum(torch.abs(m.De1.weight) + torch.abs(m.Dr1.weight)) +
                   torch.sum(torch.abs(m.De2.weight) + torch.abs(m.Dr2.weight)) + torch.sum(torch.abs(E)) +
                   torch.sum(torch.abs(Rl)))
    (total + reg).backward()
    opt.step()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_proje.py needs a CUDA device")
    torch.backends.cuda.matmul.allow_tf32 = False
    name, plimit = card()
    lines = []

    def emit(**kw):
        kw.update(gpu=name, power_limit_w=plimit)
        lines.append(kw)
        print(json.dumps(kw), flush=True)

    flush = torch.empty(64 << 20, dtype=torch.float32, device="cuda")
    kw = dict(tot_entity=N, tot_relation=R, hidden_size=K, lmbda=LMBDA, hidden_dropout=DROPOUT, device="cuda")
    rng = np.random.RandomState(0)
    h, r, t = (torch.from_numpy(rng.randint(n, size=B).astype(np.int64)).cuda() for n in (N, R, N))
    labs = []
    neg = rng.permutation(N)[:100]
    for _ in range(2):
        lab = np.zeros((B, N), np.float32)
        for b in range(B):
            lab[b, neg] = -1.0
            lab[b, rng.randint(N, size=rng.randint(1, 31))] = 1.0
        labs.append(torch.from_numpy(lab).cuda())
    nnz = int(sum((l != 0).sum().item() for l in labs))

    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    torch.manual_seed(0)
    fused = import_model("proje_pointwise")(**kw).cuda()
    cfg = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=LR, batch_size=B, tot_entity=N)
    tr = Trainer(fused, cfg)
    ev_cls, trmod.Evaluator = trmod.Evaluator, (lambda *a, **k: None)
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev_cls
    assert tr._proje
    ms = time_ms(lambda: tr.train_batch_device([h, r, t, labs[0], labs[1]]), args.reps, flush)
    emit(kernel="ProjE fused step (proje_train_step + reg_l1_dense + dense Adam x8)", case="train B=%d N=%d" % (B, N),
         ms=ms, labelled_entries=nnz, flops=3 * 2.0 * nnz * K)
    torch.manual_seed(0)
    ref = import_model("proje_pointwise")(**kw).cuda()
    opt = torch.optim.Adam(ref.parameters(), lr=LR)
    ms_ref = time_ms(lambda: dense_reference_step(ref, opt, h, r, t, labs[0], labs[1]), args.reps, flush)
    emit(kernel="reference dense formulation in torch ops (autograd + torch.optim.Adam)",
         case="train B=%d N=%d" % (B, N), ms=ms_ref, flops=2 * 3 * 2.0 * B * N * K, speedup_fused=ms_ref / ms)

    from pykg2vec_b200.evaluator import Evaluator
    model = import_model("proje_pointwise")(**kw).cuda().eval()
    ev = object.__new__(Evaluator)
    ev.model, ev.config = model, types.SimpleNamespace(device="cuda", tot_entity=N)
    ev._filter_cache, ev._workspace = {}, None
    qrng = np.random.RandomState(1)
    hs, rs, ts = qrng.randint(N, size=Q), qrng.randint(R, size=Q), qrng.randint(N, size=Q)
    ft = [np.unique(np.append(qrng.randint(N, size=20), ts[q])) for q in range(Q)]
    fh = [np.unique(np.append(qrng.randint(N, size=20), hs[q])) for q in range(Q)]
    csr = lambda rows: (np.concatenate([[0], np.cumsum([len(x) for x in rows])]).astype(np.int64),
                        np.concatenate(rows).astype(np.int64))
    ftc, fhc = csr(ft), csr(fh)
    with torch.no_grad():
        ms = time_ms(lambda: ev.rank_triples(hs, rs, ts, ftc, fhc), args.reps, flush)
    emit(kernel="Evaluator.rank_triples ProjE e2e, filtered (host ids in, ranks out)", case="eval Q=%d" % Q, ms=ms,
         flops=2 * 2.0 * Q * N * K, scored_per_s=2 * Q * N / ms * 1e3)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
