#!/usr/bin/env python
"""Projection-tail / ConvE kernel timings (NOT the driver's bench.py): ConvE on the FB15k-237
shape (N=14,541, R=237, hidden_size 200 as a 20x20 image), training batch B=128 and evaluation
batch Q=512, CUDA events, L2 flushed between repetitions.  One JSON line per measurement:

  flops  = algorithmic fp32 FLOPs of the op (2*M*N*K per GEMM use)
  frac   = flops / time / fp32 FMA-pipe peak (132 SMs x 128 lanes x 2 x SM clock, H100 SXM) — the tiled GEMM is
           bound by the fp32 pipe, not HBM (its operands are re-used on chip; ranks must be exact in
           fp32, so no tensor-core formulation in this round)
  bytes  = algorithmic HBM bytes (operands once + outputs once), GBps = bytes / time
and, for context, the same op through the torch library path the reference takes on a GPU
(matmul + add + sigmoid; topk over all N per query for ranking).

    python bench_proj.py [--reps 20] [--out gpurun_out/proj_r1.jsonl] [--one]
"""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)
from pykg2vec_b200 import _lib, import_model  # noqa: E402

N, R, K, K1 = 14541, 237, 200, 20
SM, LANES, CLOCK_GHZ = 132, 128, 1.98
FP32_PEAK_TFLOPS = SM * LANES * 2 * CLOCK_GHZ / 1e3


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    ap.add_argument("--one", action="store_true", help="a single forward + rank launch (for ncu)")
    args = ap.parse_args()
    dev = torch.device("cuda", 0)
    torch.manual_seed(0)
    model = import_model("conve")(tot_entity=N, tot_relation=R, hidden_size=K, hidden_size_1=K1, lmbda=0.1,
                                  input_dropout=0.2, feature_map_dropout=0.2, hidden_dropout=0.3).to(dev).eval()
    ent, bias = model.proj_tail_tables()
    ent, bias = ent.detach(), bias.detach()
    gen = torch.Generator(device=dev).manual_seed(1)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []

    def emit(**kw):
        kw["fp32_peak_tflops"] = FP32_PEAK_TFLOPS
        if "flops" in kw:
            kw["tflops"] = kw["flops"] / kw["ms"] / 1e9
            kw["frac"] = kw["tflops"] / FP32_PEAK_TFLOPS
        if "bytes" in kw:
            kw["GBps"] = kw["bytes"] / kw["ms"] / 1e6
        print(json.dumps(kw))
        lines.append(kw)

    for label, B in (("train B=128", 128), ("eval Q=512", 512)):
        e = torch.randint(0, N, (B,), device=dev, generator=gen)
        r = torch.randint(0, R, (B,), device=dev, generator=gen)
        tgt = torch.randint(0, N, (B,), device=dev, generator=gen)
        with torch.no_grad():
            x = model.proj_query(e, r, "tail").contiguous()
        preds = torch.empty((B, N), dtype=torch.float32, device=dev)
        if args.one:
            _lib.proj_tail_fwd(x, ent, bias, out=preds)
            _lib.proj_rank(x, ent, bias, tgt)
            torch.cuda.synchronize()
            continue
        gemm_flops = 2.0 * B * N * K
        counts = torch.zeros((B, 4), dtype=torch.int32, device=dev)
        ws = torch.empty(B * 4 + 16, dtype=torch.uint8, device=dev)
        for tile, tname in ((None, "auto"), ("0", "64x64"), ("1", "64x128"), ("2", "128x128")):
            if tile is None:
                os.environ.pop("KGE_PROJ_TILE", None)
            else:
                os.environ["KGE_PROJ_TILE"] = tile      # read by the library at every call
            ms = time_ms(lambda: _lib.proj_tail_fwd(x, ent, bias, out=preds), args.reps, flush)
            emit(kernel="proj_tail_fwd", tile=tname, case=label, ms=ms, flops=gemm_flops,
                 bytes=(B * K + N * K + N + B * N) * 4)
            ms = time_ms(lambda: _lib.proj_rank(x, ent, bias, tgt, None, 0, counts, ws), args.reps, flush)
            emit(kernel="proj_rank (1 direction, raw)", tile=tname, case=label, ms=ms, flops=gemm_flops,
                 bytes=(B * K + N * K + N) * 4, scored_per_s=B * N / ms * 1e3)
        os.environ.pop("KGE_PROJ_TILE", None)
        ms = time_ms(lambda: torch.sigmoid(torch.addmm(bias, x, ent.T)), args.reps, flush)
        emit(kernel="torch addmm+sigmoid (library)", case=label, ms=ms, flops=gemm_flops)
        ms = time_ms(lambda: torch.topk(-torch.sigmoid(torch.addmm(bias, x, ent.T)), k=N), max(args.reps // 4, 3), flush)
        emit(kernel="torch addmm+sigmoid+topk(N) (library, batched)", case=label, ms=ms, scored_per_s=B * N / ms * 1e3)
        labels = (torch.rand((B, N), device=dev, generator=gen) < 0.01).float()
        ms = time_ms(lambda: _lib.proj_bce(preds, labels, 0.9, 1.0 / N, 1.0), args.reps, flush)
        emit(kernel="proj_bce (value + grad)", case=label, ms=ms, bytes=3 * B * N * 4)
        gp = torch.randn((B, N), device=dev, generator=gen) * 1e-6
        gx, ge, gb = torch.zeros_like(x), torch.zeros_like(ent), torch.zeros(N, device=dev)
        ms = time_ms(lambda: _lib.proj_tail_bwd(gp, preds, x, ent, gx, ge, gb), args.reps, flush)
        emit(kernel="proj_tail_bwd (grad_x + grad_ent + grad_bias)", case=label, ms=ms, flops=2 * gemm_flops,
             bytes=(4 * B * N + 2 * N * K + 2 * B * K) * 4)
        with torch.no_grad():
            ms = time_ms(lambda: _lib.conve_trunk_fwd(model, e, r), args.reps, flush)
            F = model.fc.in_features
            emit(kernel="conve_trunk_fwd (feature kernel + Linear GEMM)", case=label, ms=ms,
                 flops=2.0 * B * F * K + 2.0 * B * F * 9)
            ms = time_ms(lambda: model._trunk_layers(e, r), args.reps, flush)
            emit(kernel="torch trunk (cuDNN/cuBLAS library layers)", case=label, ms=ms)
    if not args.one:
        # end to end: Evaluator.rank_triples on host ids (H2D + trunk x2 + rank x2 + D2H), Q=512
        import types
        from pykg2vec_b200.evaluator import Evaluator
        ev = object.__new__(Evaluator)
        ev.model, ev.config = model, types.SimpleNamespace(device="cuda", tot_entity=N)
        ev._filter_cache, ev._workspace = {}, None
        rng = np.random.RandomState(0)
        hs, rs, ts = rng.randint(N, size=512), rng.randint(R, size=512), rng.randint(N, size=512)
        with torch.no_grad():
            ms = time_ms(lambda: ev.rank_triples(hs, rs, ts), args.reps, flush)
        emit(kernel="Evaluator.rank_triples ConvE e2e (host ids in, ranks out)", case="eval Q=512", ms=ms,
             scored_per_s=2 * 512 * N / ms * 1e3)
        # training step end to end (adam, B=128, label smoothing 0.1): the reference's data path (ids +
        # two dense [B,N] label matrices from the host every step, generator.py:160-236) vs label rows
        # built on the device from CSRs (pykg2vec_b200.generator.Generator)
        from pykg2vec_b200.generator import Generator
        from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
        from pykg2vec_b200.trainer import Trainer
        kg = SyntheticKnowledgeGraph.shaped_like("fb15k_237", scale=0.2)
        cfg = SyntheticConfig(kg, device="cuda", optimizer="adam", learning_rate=0.003, batch_size=128, neg_rate=0,
                              hidden_size=K, hidden_size_1=K1, lmbda=0.1, input_dropout=0.2, feature_map_dropout=0.2,
                              hidden_dropout=0.3, label_smoothing=0.1)
        tmodel = import_model("conve")(**cfg.__dict__)
        tr = Trainer(tmodel, cfg)
        tr.build_model()
        gen = Generator(tmodel, cfg, seed=0)
        gen.start_one_epoch(10 ** 6)
        ms = time_ms(lambda: tr.train_batch_device(next(gen)), args.reps, flush)
        emit(kernel="ConvE train step, device label rows (Generator -> train_batch_device)", case="train B=128", ms=ms,
             scored_per_s=2 * 128 * N / ms * 1e3)
        hb, rb, tb, lt, lh = (v.cpu() for v in next(gen))
        host = [hb.numpy(), rb.numpy(), tb.numpy(), lt, lh]
        ms = time_ms(lambda: tr.train_batch(host), args.reps, flush)
        emit(kernel="ConvE train step, host dense labels (reference data path: 2*B*N floats H2D)", case="train B=128",
             ms=ms, scored_per_s=2 * 128 * N / ms * 1e3, h2d_bytes=tr.last_h2d_bytes)
    if args.out:
        with open(args.out, "w") as f:
            for l in lines:
                f.write(json.dumps(l) + "\n")


if __name__ == "__main__":
    main()
