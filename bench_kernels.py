#!/usr/bin/env python
"""Per-kernel roofline sweep (NOT the driver's bench.py): fused gather+score forward /
backward / fused train step on tables far larger than the 50 MB L2, random ids, so the row
gathers really come from HBM.  Prints one JSON line per case:

    achieved GB/s = ALGORITHMIC bytes (SURVEY.md 8d: rows*d*4 + 24 B ids + 4 B score per triple;
                    x4 for forward+backward) / CUDA-event time,   frac = achieved / measured peak.

    python bench_kernels.py [--reps 20] [--out gpurun_out/kernels_r1.jsonl]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from bench import peaks  # noqa: E402
from pykg2vec_b200 import _lib  # noqa: E402

ROWS = {"transe": 3, "distmult": 3, "transh": 4, "rotate": 5, "complex": 6, "transd": 6}
NTAB = {"transe": ["e", "r"], "distmult": ["e", "r"], "transh": ["e", "r", "r"], "rotate": ["e", "e", "r"],
        "complex": ["e", "e", "r", "r"], "transd": ["e", "r", "e", "r"]}

CASES = [
    # name, N, R, d, n triples, l1
    ("transe", 1_000_000, 1000, 200, 4_000_000, False),
    ("transe", 4_000_000, 1000, 50, 8_000_000, True),
    ("distmult", 1_000_000, 1000, 200, 4_000_000, False),
    ("complex", 500_000, 1000, 200, 2_000_000, False),
    ("complex", 250_000, 1000, 500, 1_000_000, False),
    ("rotate", 200_000, 1000, 1000, 400_000, False),
    ("transh", 1_000_000, 1000, 200, 2_000_000, False),
    ("transd", 500_000, 1000, 200, 2_000_000, False),
]


def time_ms(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(reps):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--only", default=None)
    args = ap.parse_args()
    peak, src, _ = peaks()
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev).manual_seed(0)
    lines = []
    for name, N, R, d, n, l1 in CASES:
        if args.only and args.only != name:
            continue
        tabs = []
        for kind in NTAB[name]:
            rows = N if kind == "e" else R
            tabs.append((torch.rand((rows, d), device=dev, generator=gen) - 0.5) * 0.2)
        desc = _lib.ModelDesc(name, tabs, d, l1_flag=l1, margin=24.0 if name == "rotate" else 0.0,
                              phase_scale=float(np.pi / ((24.0 + 2) / d)) if name == "rotate" else 0.0)
        h = torch.randint(0, N, (n,), device=dev, generator=gen)
        r = torch.randint(0, R, (n,), device=dev, generator=gen)
        t = torch.randint(0, N, (n,), device=dev, generator=gen)
        out = torch.empty(n, dtype=torch.float32, device=dev)
        fwd_bytes = n * (ROWS[name] * d * 4 + 28)
        ms = time_ms(lambda: _lib.score_fwd(desc, h, r, t, out=out), args.reps)
        line = {"kernel": "score_fwd", "model": name, "N": N, "d": d, "n": n, "ms": ms,
                "algorithmic_bytes": fwd_bytes, "achieved_GBps": fwd_bytes / ms / 1e6, "peak_GBps": peak,
                "frac": fwd_bytes / ms / 1e6 / peak, "peak_source": src, "triples_per_s": n / ms * 1e3}
        print(json.dumps(line))
        lines.append(line)
        # backward into dense grad tables (rows re-read + row gradients read-modify-written)
        nb = n // 4
        grads = [torch.zeros_like(x) for x in tabs]
        g = torch.randn(nb, device=dev, generator=gen)
        bwd_bytes = nb * (ROWS[name] * d * 4 * 3 + 28)
        ms = time_ms(lambda: _lib.score_bwd(desc, h[:nb], r[:nb], t[:nb], g, grads), max(args.reps // 4, 3))
        line = {"kernel": "score_bwd", "model": name, "N": N, "d": d, "n": nb, "ms": ms,
                "algorithmic_bytes": bwd_bytes, "achieved_GBps": bwd_bytes / ms / 1e6, "peak_GBps": peak,
                "frac": bwd_bytes / ms / 1e6 / peak, "peak_source": src, "triples_per_s": nb / ms * 1e3}
        print(json.dumps(line))
        lines.append(line)
        del grads, tabs, desc
        torch.cuda.empty_cache()
    if args.out:
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
