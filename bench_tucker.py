#!/usr/bin/env python
"""TuckER at the FB15k-237 shape (N = 14,541, R = 237, d1 = d2 = 200): the kernel path against the torch layers.

  training   B = 128, dropouts 0.3 / 0.4 / 0.5, Adam: Trainer's fused step (kge_tucker_*: one core matrix per distinct
             relation) vs train_step_projection + loss.backward() + torch.optim.Adam on TuckER._trunk_layers (one
             matrix per sample, the reference's formulation)
  evaluation one batch of Q = 512 queries, both directions: proj_query with per-call core matrices vs _trunk_layers

Both arms of a pair run in one process, alternating, `--rounds` times; each timing is a device-event window of
`--iters` warmed iterations (sized to last well over a second).  Reported per arm: the median and the spread over
the rounds, torch.cuda.max_memory_allocated of one iteration above the standing allocations, the bytes and FLOPs the
two formulations need counted from the shapes, the card's name and power limit (queried, never set), and the largest
difference of the two arms' outputs on the same seeded inputs.  Without a GPU it exits with an error.

    python bench_tucker.py [--iters 1500] [--rounds 3]
"""
import argparse
import json
import subprocess
import sys
import types

import numpy as np
import torch

N, R, D, B, Q = 14541, 237, 200, 128, 512
DROPS = (0.3, 0.4, 0.5)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:   # the query is informative only
        out = "unknown (%s)" % exc
    return out


def trainer(fused, drops):
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    torch.manual_seed(0)
    m = import_model("tucker")(tot_entity=N, tot_relation=R, ent_hidden_size=D, rel_hidden_size=D, lmbda=0.0,
                               input_dropout=drops[0], hidden_dropout1=drops[1], hidden_dropout2=drops[2],
                               kge_trunk=fused).cuda()
    cfg = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=1e-3, fused_step=fused,
                                label_smoothing=0.1, tot_entity=N, batch_size=B, knowledge_graph=None)
    tr = Trainer(m, cfg)
    ev, trmod.Evaluator = trmod.Evaluator, (lambda *a, **k: None)
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev
    return tr


def window(fn, iters):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b) / iters


def peak(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def compare(arms, iters, rounds):
    for fn in arms.values():
        for _ in range(10):
            fn()
    times = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            times[k].append(window(fn, iters))
    return {k: {"ms_median": float(np.median(v)), "ms_min": min(v), "ms_max": max(v), "peak_bytes": peak(arms[k])}
            for k, v in times.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=1500)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_tucker.py needs a CUDA device")
    gen = torch.Generator("cuda").manual_seed(1)
    ids = [torch.randint(N, (B,), device="cuda", generator=gen), torch.randint(R, (B,), device="cuda", generator=gen),
           torch.randint(N, (B,), device="cuda", generator=gen)]
    labels = [(torch.rand(B, N, device="cuda", generator=gen) < 0.001).float() for _ in range(2)]
    batch = ids + labels
    U = int(torch.unique(ids[1]).numel())
    res = {"card": card(), "shape": {"N": N, "R": R, "d1": D, "d2": D, "B": B, "Q": Q, "distinct_relations_in_batch": U},
           "iters": args.iters, "rounds": args.rounds}
    # what the two formulations must move / compute per training step (both directions, forward only), from shapes
    res["counted"] = {
        "per_sample": {"matrix_bytes": 2 * B * D * D * 4, "build_flops": 2 * 2 * B * D * D * D},
        "per_relation": {"matrix_bytes": U * D * D * 4, "build_flops": 2 * U * D * D * D},
    }
    # same seeded inputs, dropouts 0: the two arms compute the same step
    fa, fb = trainer(True, (0, 0, 0)), trainer(False, (0, 0, 0))
    la, lb = float(fa.train_batch_device(batch)), float(fb.train_batch_device(batch))
    res["train_check"] = {"loss_fused": la, "loss_layers": lb, "max_abs_diff_tables": max(
        float((p.weight.detach() - q.weight.detach()).abs().max()) for p, q in zip(fa.model.parameter_list, fb.model.parameter_list))}
    del fa, fb
    a, b = trainer(True, DROPS), trainer(False, DROPS)
    res["train"] = compare({"fused_kernels": lambda: a.train_batch_device(batch),
                            "autograd_torch_layers": lambda: b.train_batch_device(batch)}, args.iters, args.rounds)
    m, ml = a.model.eval(), b.model.eval()
    ml.load_state_dict(m.state_dict())
    qh = torch.randint(N, (Q,), device="cuda", generator=gen)
    qr = torch.randint(R, (Q,), device="cuda", generator=gen)
    qt = torch.randint(N, (Q,), device="cuda", generator=gen)

    def eval_kernels():
        cores = m.proj_query_cores(qr)
        return m.proj_query(qh, qr, cores=cores), m.proj_query(qt, qr, cores=cores)

    def eval_layers():
        return ml.proj_query(qh, qr), ml.proj_query(qt, qr)

    with torch.no_grad():
        res["eval_check"] = {"max_abs_diff_x": max(float((u - v).abs().max()) for u, v in zip(eval_kernels(), eval_layers()))}
        res["eval"] = compare({"per_call_cores": eval_kernels, "torch_layers": eval_layers}, args.iters, args.rounds)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
