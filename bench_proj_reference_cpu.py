#!/usr/bin/env python
"""CPU timing of the UNMODIFIED reference ConvE (pykg2vec/models/projection.py:12-125) on the workload
bench_proj.py times on the GPU: FB15k-237 shape (N=14,541, R=237, hidden_size 200 as 20x20),
  * evaluation as the reference runs it (evaluator.py:309-334): per test triple one predict_tail_rank and
    one predict_head_rank — a [1,N] forward + topk(N) each — and the Python rank walk of MetricCalculator;
  * one training step (trainer.py:159-174,298-299): both directions, multi_class_bce with label smoothing,
    backward, adam, batch 128, dense [128,N] label matrices.
Needs the reference package installed (baseline/install_ref.sh) and runs on host cores (stated in the output):
the numbers are an indication beside bench_proj.py's, not a bench value.

    python bench_proj_reference_cpu.py [--queries 40] [--steps 5] [--out FILE.json]
"""
import argparse
import json
import os
import sys
import time
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
import make_golden as mg  # noqa: E402  (import stubs + /root/reference on sys.path)

from pykg2vec.models import projection as ref_projection  # noqa: E402
from pykg2vec.utils.criterion import Criterion  # noqa: E402
from pykg2vec.utils.evaluator import Evaluator, MetricCalculator  # noqa: E402

N, R, K, K1 = 14541, 237, 200, 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--queries", type=int, default=40)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    cores = os.cpu_count()
    torch.set_num_threads(cores)
    torch.manual_seed(0)
    m = ref_projection.ConvE(tot_entity=N, tot_relation=R, hidden_size=K, hidden_size_1=K1, lmbda=0.1,
                             input_dropout=0.2, feature_map_dropout=0.2, hidden_dropout=0.3)
    rng = np.random.RandomState(0)
    # ---- evaluation, exactly the reference's per-triple path --------------------------------------
    ev = object.__new__(Evaluator)
    ev.model = m
    ev.config = types.SimpleNamespace(tot_entity=N, device="cpu")
    mc = object.__new__(MetricCalculator)
    q = [(int(rng.randint(N)), int(rng.randint(R)), int(rng.randint(N))) for _ in range(args.queries + 3)]
    mc.hr_t = {(h, r): {t} for h, r, t in q}
    mc.tr_h = {(t, r): {h} for h, r, t in q}
    m.eval()
    times = []
    with torch.no_grad():
        for i, (h, r, t) in enumerate(q):
            t0 = time.perf_counter()
            hrank = ev.test_head_rank(torch.LongTensor([r]), torch.LongTensor([t]), N).numpy()
            trank = ev.test_tail_rank(torch.LongTensor([h]), torch.LongTensor([r]), N).numpy()
            mc.get_tail_rank(trank, h, r, t)
            mc.get_head_rank(hrank, h, r, t)
            if i >= 3:
                times.append(time.perf_counter() - t0)
    ms_q = float(np.mean(times)) * 1e3
    # ---- one training step ---------------------------------------------------------------------------
    m.train()
    opt = torch.optim.Adam(m.parameters(), lr=0.003)
    B = 128
    h, r, t = (torch.from_numpy(rng.randint(n, size=B)) for n in (N, R, N))
    hr_t = torch.zeros(B, N)
    tr_h = torch.zeros(B, N)
    hr_t[torch.arange(B), t] = 1.0
    tr_h[torch.arange(B), h] = 1.0
    st = []
    for i in range(args.steps + 2):
        t0 = time.perf_counter()
        opt.zero_grad()
        loss = Criterion.multi_class_bce(m(t, r, direction="head"), m(h, r, direction="tail"), tr_h, hr_t, 0.1, N)
        loss.backward()
        opt.step()
        if i >= 2:
            st.append(time.perf_counter() - t0)
    ms_step = float(np.mean(st)) * 1e3
    line = {"what": "reference ConvE on CPU (unmodified pykg2vec classes, torch %s)" % torch.__version__,
            "where": "build container host cores (NOT the GPU box)", "cores": cores, "N": N, "R": R, "hidden_size": K,
            "eval_ms_per_test_triple": ms_q, "eval_scored_per_s": 2.0 * N / ms_q * 1e3, "eval_queries_timed": len(times),
            "train_step_ms_B128": ms_step, "train_scored_per_s": 2.0 * B * N / ms_step * 1e3, "train_steps_timed": len(st)}
    print(json.dumps(line))
    if args.out:
        with open(args.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
