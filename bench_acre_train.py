#!/usr/bin/env python
"""AcrE's training step at the FB15k-237 shape (N = 14,541, R = 237, B = 128, Adam at lr 1e-4, dropouts 0.3 / 0.2 /
0.5 for input / feature map / hidden, label smoothing 0.1) in one of two configurations (--config): serial (C = 32,
atrous 1/2/2, conv bias: the reference's AcrE.yaml) or parallel (C = 9, atrous 1/2/2, conv bias: the CLI defaults).
Three arms on the same batch:

  fused_kernels          Trainer's fused step: kge_acre_train_fwd over both directions -> tail + BCE ->
                         kge_acre_train_bwd -> one dense Adam sweep per parameter tensor
  autograd_kernels       train_step_projection + loss.backward() + torch.optim.Adam, trunk = AcreTrunkFunction
  autograd_torch_layers  the same on AcrE._trunk_layers (the reference's torch layers, kge_trunk = False)

The arms run in one process, alternating, `--rounds` times; each timing is a device-event window of `--iters` warmed
steps.  Reported per arm: the median and the spread over the rounds and torch.cuda.max_memory_allocated of one step
above the standing tensors.  Also: the FLOPs of the step counted from the shapes, the card's name and power limit
(queried, never set), and the largest difference of the loss and the tables after one step of the fused and the
torch-layer arms on the same seeded inputs with dropouts 0.  Without a GPU it exits with an error.

    python bench_acre_train.py [--config serial|parallel] [--iters 300] [--rounds 3]
"""
import argparse
import json
import subprocess
import sys
import types

import numpy as np
import torch

N, R, B, K = 14541, 237, 128, 200
DROPS = (0.3, 0.2, 0.5)   # input, feature map, hidden
CONFIGS = {"serial": ("serial", 32, (1, 2, 2), True), "parallel": ("parallel", 9, (1, 2, 2), True)}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:   # the query is informative only
        out = "unknown (%s)" % exc
    return out


def trainer(arm, config, drops):
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    way, C, atrous, bias = config
    torch.manual_seed(0)
    m = import_model("acre")(tot_entity=N, tot_relation=R, hidden_size=K, input_dropout=drops[0],
                             feature_map_dropout=drops[1], hidden_dropout=drops[2], in_channels=C, way=way,
                             first_atrous=atrous[0], second_atrous=atrous[1], third_atrous=atrous[2], acre_bias=bias,
                             kge_trunk=arm != "autograd_torch_layers").cuda()
    cfg = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=1e-4,
                                fused_step=arm == "fused_kernels", label_smoothing=0.1, tot_entity=N, batch_size=B,
                                knowledge_graph=None)
    tr = Trainer(m, cfg)
    ev, trmod.Evaluator = trmod.Evaluator, (lambda *a, **k: None)
    try:
        tr.build_model()
    finally:
        trmod.Evaluator = ev
    assert tr._acre == (arm == "fused_kernels")
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


def counted_gflop(config):
    """per step, both directions: forward + the two gradient products of the tail, the Linear layer, the three
    convolutions (the per-query weight gradient and the transposed convolution) and, in the parallel way, W_gate_e"""
    way, C, _, _ = config
    Fw = C * 400
    per = {"tail": 2 * B * N * K, "linear": 2 * B * Fw * K}
    if way == "serial":
        per["conv"] = 2 * B * 400 * 9 * (C + 2 * C * C)
    else:
        per["conv"] = 2 * B * 400 * 9 * 3 * C
        per["gate"] = 2 * B * C * 1600 * 400
    out = {k + "_per_step": 3 * 2 * v / 1e9 for k, v in per.items()}
    out["step"] = 3 * 2 * sum(per.values()) / 1e9
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="serial", choices=sorted(CONFIGS))
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    config = CONFIGS[args.config]
    if not torch.cuda.is_available():
        sys.exit("bench_acre_train.py needs a CUDA device")
    gen = torch.Generator("cuda").manual_seed(1)
    ids = [torch.randint(N, (B,), device="cuda", generator=gen), torch.randint(R, (B,), device="cuda", generator=gen),
           torch.randint(N, (B,), device="cuda", generator=gen)]
    labels = [(torch.rand(B, N, device="cuda", generator=gen) < 0.001).float() for _ in range(2)]
    batch = ids + labels
    way, C, atrous, bias = config
    res = {"card": card(), "shape": {"N": N, "R": R, "B": B, "way": way, "in_channels": C, "atrous": list(atrous),
                                     "acre_bias": bias, "features": C * 400, "dropouts": DROPS},
           "iters": args.iters, "rounds": args.rounds, "counted_gflop": counted_gflop(config)}
    # same seeded inputs, dropouts 0: one step of the fused and the torch-layer arms
    fa, fb = trainer("fused_kernels", config, (0, 0, 0)), trainer("autograd_torch_layers", config, (0, 0, 0))
    la, lb = float(fa.train_batch_device(batch)), float(fb.train_batch_device(batch))
    res["train_check"] = {"loss_fused": la, "loss_layers": lb, "abs_diff_loss": abs(la - lb), "max_abs_diff_tables": max(
        float((p.detach() - q.detach()).abs().max()) for p, q in zip(fa.model.parameters(), fb.model.parameters()))}
    del fa, fb
    trs = {arm: trainer(arm, config, DROPS) for arm in ("fused_kernels", "autograd_kernels", "autograd_torch_layers")}
    arms = {arm: (lambda tr=tr: tr.train_batch_device(batch)) for arm, tr in trs.items()}
    for fn in arms.values():
        for _ in range(10):
            fn()
    times = {k: [] for k in arms}
    for _ in range(args.rounds):
        for k, fn in arms.items():
            times[k].append(window(fn, args.iters))
    res["train"] = {k: {"ms_median": float(np.median(v)), "ms_min": min(v), "ms_max": max(v),
                        "peak_bytes": peak(arms[k])} for k, v in times.items()}
    ref = res["train"]["autograd_torch_layers"]["ms_median"]
    res["speedup_vs_torch_layers"] = {k: ref / v["ms_median"] for k, v in res["train"].items()}
    res["step_tflops"] = {k: res["counted_gflop"]["step"] / v["ms_median"] for k, v in res["train"].items()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
