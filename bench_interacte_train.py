#!/usr/bin/env python
"""InteractE's training step at the FB15k-237 shape (N = 14,541, R = 237, B = 128, Adam at lr 1e-4, dropouts
0.2 / 0.5 / 0.3, label smoothing 0.1: the reference's InteractE.yaml) at one of its three geometries (--geom P,F,ks;
the image is always 20 x 10 per half): three arms on the same batch.

  fused_kernels          Trainer's fused step: kge_interacte_train_fwd over both directions -> tail + BCE ->
                         kge_interacte_train_bwd -> one dense Adam sweep per parameter tensor
  autograd_kernels       train_step_projection + loss.backward() + torch.optim.Adam, trunk = InteracteTrunkFunction
  autograd_torch_layers  the same on InteractE._trunk_layers (the reference's torch layers, kge_trunk = False)

The arms run in one process, alternating, `--rounds` times; each timing is a device-event window of `--iters` warmed
steps.  Reported per arm: the median and the spread over the rounds and torch.cuda.max_memory_allocated of one step
above the standing tensors.  Also: the FLOPs of the step counted from the shapes, the card's name and power limit
(queried, never set), and the largest difference of the loss and the tables after one step of the fused and the
torch-layer arms on the same seeded inputs with dropouts 0.  Without a GPU it exits with an error.

    python bench_interacte_train.py [--geom 1,96,9] [--iters 300] [--rounds 3]
"""
import argparse
import json
import subprocess
import sys
import types

import numpy as np
import torch

N, R, B, RH, RW = 14541, 237, 128, 20, 10
K = RH * RW
DROPS = (0.2, 0.5, 0.3)   # input, feature map, hidden
GEOMS = ((1, 96, 9), (2, 96, 11), (4, 64, 7))


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as exc:   # the query is informative only
        out = "unknown (%s)" % exc
    return out


def trainer(arm, geom, drops):
    from pykg2vec_b200 import import_model
    from pykg2vec_b200.trainer import Trainer
    import pykg2vec_b200.trainer as trmod
    P, F, ks = geom
    torch.manual_seed(0)
    np.random.seed(0)   # the chequer permutation
    m = import_model("interacte")(tot_entity=N, tot_relation=R, hidden_size=K, input_dropout=drops[0],
                                  feature_map_dropout=drops[1], hidden_dropout=drops[2], feature_permutation=P,
                                  num_filters=F, kernel_size=ks, reshape_height=RH, reshape_width=RW, device="cuda",
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
    assert tr._interacte == (arm == "fused_kernels")
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


def counted_gflop(geom):
    """per step, both directions: forward + the two gradient products of the tail, the Linear layer and the circular
    convolution (the per-query filter gradient and the transposed convolution)"""
    P, F, ks = geom
    Fw = P * F * 2 * K
    per = {"tail": 2 * B * N * K, "linear": 2 * B * Fw * K, "conv": 2 * B * Fw * ks * ks}
    out = {k + "_per_step": 3 * 2 * v / 1e9 for k, v in per.items()}
    out["step"] = 3 * 2 * sum(per.values()) / 1e9
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--geom", default="1,96,9", help="P,F,ks: one of %s" % (GEOMS,))
    ap.add_argument("--iters", type=int, default=300)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    geom = tuple(int(v) for v in args.geom.split(","))
    if geom not in GEOMS:
        sys.exit("--geom must be one of %s" % (GEOMS,))
    if not torch.cuda.is_available():
        sys.exit("bench_interacte_train.py needs a CUDA device")
    gen = torch.Generator("cuda").manual_seed(1)
    ids = [torch.randint(N, (B,), device="cuda", generator=gen), torch.randint(R, (B,), device="cuda", generator=gen),
           torch.randint(N, (B,), device="cuda", generator=gen)]
    labels = [(torch.rand(B, N, device="cuda", generator=gen) < 0.001).float() for _ in range(2)]
    batch = ids + labels
    P, F, ks = geom
    res = {"card": card(), "shape": {"N": N, "R": R, "B": B, "P": P, "F": F, "ks": ks, "image": [2 * RW, RH],
                                     "features": P * F * 2 * K, "dropouts": DROPS},
           "iters": args.iters, "rounds": args.rounds, "counted_gflop": counted_gflop(geom)}
    # same seeded inputs, dropouts 0: one step of the fused and the torch-layer arms
    fa, fb = trainer("fused_kernels", geom, (0, 0, 0)), trainer("autograd_torch_layers", geom, (0, 0, 0))
    la, lb = float(fa.train_batch_device(batch)), float(fb.train_batch_device(batch))
    res["train_check"] = {"loss_fused": la, "loss_layers": lb, "abs_diff_loss": abs(la - lb), "max_abs_diff_tables": max(
        float((p.detach() - q.detach()).abs().max()) for p, q in zip(fa.model.parameters(), fb.model.parameters()))}
    del fa, fb
    trs = {arm: trainer(arm, geom, DROPS) for arm in ("fused_kernels", "autograd_kernels", "autograd_torch_layers")}
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
