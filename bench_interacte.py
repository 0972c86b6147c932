#!/usr/bin/env python
"""InteractE timings (NOT bench.py, which times the flagship workload) on the FB15k-237 shape
(N=14,541, R=237, feature_permutation 1, num_filters 96, kernel_size 9, reshape 20 x 10, hyperparams/InteractE.yaml),
CUDA events, L2 flushed before every repetition.  One JSON line per measurement, each carrying the card's name and
power limit read in the same run (nvidia-smi --query-gpu, read only):

  trunk        kge_interacte_trunk_fwd (feature kernel + Linear GEMM + bn2/ReLU) against the reference's torch
               layers on the same device (gather + permutation, circular padding, cuDNN grouped conv with TF32
               off, cuBLAS Linear), Q = 512, tail and head direction (InteractE runs the same function on (h, r)
               and (t, r)); the feature kernel and the Linear GEMM + combine are also timed on their own
  rank e2e     Evaluator.rank_triples for 512 filtered queries: host ids in, host ranks out
  train step   one Trainer.train_batch at B = 128 (adam, label smoothing 0.1, host dense label rows)

  flops        algorithmic fp32 FLOPs from the shapes: the conv 2*ks^2*Q*P*F*H*W (3.2 GFLOP at Q = 512), the
               Linear layer 2*Q*P*F*H*W*k (7.9 GFLOP at Q = 512).
Before timing, the script checks that both trunk paths give the same ranks (kernel trunk vs torch layers,
through the same kge_proj_rank): equal, except that a query may differ by the candidates whose prediction is
within the two paths' largest prediction difference of its target's (the trunks round differently; the
check line reports how many queries are equal).  Inputs are fixed-seed.

    python bench_interacte.py [--reps 20] [--out results/interacte.jsonl]
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

N, R, Q, B = 14541, 237, 512, 128
P, NF, KS, RH, RW = 1, 96, 9, 20, 10
D = RH * RW                      # k = 200
H, W = 2 * RW, RH
F = P * NF * H * W               # 38,400 features per query


def card():
    """(name, power limit) of GPU 0 as nvidia-smi reports them: the limit in W, or nvidia-smi's own text when it
    gives no number (e.g. "[N/A]")"""
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,enforced.power.limit",
                              "--format=csv,noheader,nounits", "-i", "0"],
                             capture_output=True, text=True, timeout=60).stdout.strip()
    except Exception as exc:   # the timings stand without it, but say why the fields are missing
        return "unknown (%s)" % exc, None
    fields = [f.strip() for f in out.split(",")]
    name, limits = fields[0], fields[1:]
    for v in limits:
        try:
            return name, float(v)
        except ValueError:
            pass
    return name, " / ".join(limits) or None


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
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_interacte.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, power = card()
    torch.manual_seed(0)
    np.random.seed(0)
    kw = dict(tot_entity=N, tot_relation=R, hidden_size=D, input_dropout=0.2, hidden_dropout=0.3,
              feature_map_dropout=0.5, feature_permutation=P, num_filters=NF, kernel_size=KS, reshape_height=RH,
              reshape_width=RW, device="cuda")
    model = import_model("interacte")(**kw)
    with torch.no_grad():   # non-trivial BatchNorm statistics and bias, as a trained model has
        for bn in (model.bn0, model.bn1, model.bn2):
            bn.running_mean.normal_(0.0, 0.2)
            bn.running_var.uniform_(0.5, 1.5)
        model.bias.normal_(0.0, 0.3)
    model = model.to(dev).eval()
    ent, bias = (t.detach() for t in model.proj_tail_tables())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    lines = []

    def emit(**kw):
        kw.update(gpu=name, power_limit_w=power)
        if "flops" in kw:
            kw["tflops"] = kw["flops"] / kw["ms"] / 1e9
        print(json.dumps(kw), flush=True)
        lines.append(kw)

    rng = np.random.RandomState(0)
    hs, rs, ts = rng.randint(N, size=Q), rng.randint(R, size=Q), rng.randint(N, size=Q)
    h, r, t = (torch.from_numpy(a).to(dev) for a in (hs, rs, ts))
    conv_flops, fc_flops = 2.0 * KS * KS * Q * F, 2.0 * Q * F * D
    trunk_flops = conv_flops + fc_flops
    ws = torch.empty(_lib.interacte_trunk_workspace_bytes(P, NF, KS, RH, RW, R, Q), dtype=torch.uint8, device=dev)
    perm = model.chequer_perm.to(dev)
    with torch.no_grad():
        # both trunk paths rank alike (same tail kernel, exact counts) before anything is timed.  The two trunks
        # round differently (~1e-6), so a query may only differ by candidates whose prediction lies within the
        # largest prediction difference of the two paths from its target's
        for direction, e, tgt in (("tail", h, t), ("head", t, h)):
            xk = _lib.interacte_trunk_fwd(model, e, r, workspace=ws, perm=perm)
            xt = model._trunk_layers(e, r).contiguous()
            ck = _lib.proj_rank(xk, ent, bias, tgt)[:, 0]
            ct = _lib.proj_rank(xt, ent, bias, tgt)[:, 0]
            pk, pt = _lib.proj_tail_fwd(xk, ent, bias), _lib.proj_tail_fwd(xt, ent, bias)
            band = 2 * (pk - pt).abs().max(1, keepdim=True).values
            near = ((pk - pk.gather(1, tgt[:, None])).abs() <= band).sum(1) - 1
            if ((ck - ct).abs() > near).any():
                raise SystemExit("kernel and torch-layer trunks rank %s queries differently beyond near ties" % direction)
            emit(check="ranks of kernel trunk vs torch layers", direction=direction, queries=Q,
                 equal=int((ck == ct).sum()), differ_within_near_ties=int((ck != ct).sum()),
                 max_abs_x_diff=float((xk - xt).abs().max()))
        for direction, e in (("tail", h), ("head", t)):
            ms = time_ms(lambda: _lib.interacte_trunk_fwd(model, e, r, workspace=ws, perm=perm), args.reps, flush)
            emit(kernel="kge_interacte_trunk_fwd (features + Linear + bn2/relu)", case="eval Q=%d" % Q,
                 direction=direction, ms=ms, flops=trunk_flops)
            ms = time_ms(lambda: model._trunk_layers(e, r), args.reps, flush)
            emit(kernel="torch trunk (reference layers: cuDNN grouped conv, cuBLAS Linear)", case="eval Q=%d" % Q,
                 direction=direction, ms=ms, flops=trunk_flops)
        # the conv / Linear split: the whole trunk profiled once, device time per kernel
        with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
            for _ in range(args.reps):
                _lib.interacte_trunk_fwd(model, h, r, workspace=ws, perm=perm)
            torch.cuda.synchronize()
        split = {}
        for ev_ in prof.key_averages():
            for tag in ("interacte_feature_kernel", "proj_gemm_kernel", "hyper_fc_combine_kernel"):
                if tag in ev_.key:
                    split[tag] = split.get(tag, 0.0) + getattr(ev_, "device_time_total", 0.0) / 1e3 / args.reps
        emit(kernel="interacte_feature_kernel (gather + perm + bn0 + circular conv + bn1 + relu)",
             case="eval Q=%d, profiled, L2 warm" % Q, ms=split.get("interacte_feature_kernel", float("nan")),
             flops=conv_flops)
        emit(kernel="Linear GEMM + bn2/relu combine", case="eval Q=%d, profiled, L2 warm" % Q,
             ms=split.get("proj_gemm_kernel", float("nan")) + split.get("hyper_fc_combine_kernel", float("nan")),
             flops=fc_flops)
        # end to end: Evaluator.rank_triples on host ids with filters (H2D + trunk x2 + rank x2 + D2H)
        from pykg2vec_b200.evaluator import Evaluator
        ev = object.__new__(Evaluator)
        ev.model, ev.config = model, types.SimpleNamespace(device="cuda", tot_entity=N)
        ev._filter_cache, ev._workspace = {}, None
        frng = np.random.RandomState(1)
        ft, fh = [], []
        for q in range(Q):
            ft.append(np.unique(np.append(frng.randint(N, size=20), ts[q])))
            fh.append(np.unique(np.append(frng.randint(N, size=20), hs[q])))
        csr = lambda rows: (np.concatenate([[0], np.cumsum([len(x) for x in rows])]).astype(np.int64),
                            np.concatenate(rows).astype(np.int64))
        ftc, fhc = csr(ft), csr(fh)
        ms = time_ms(lambda: ev.rank_triples(hs, rs, ts, ftc, fhc), args.reps, flush)
        emit(kernel="Evaluator.rank_triples InteractE e2e, filtered (host ids in, ranks out)", case="eval Q=%d" % Q, ms=ms,
             flops=2 * trunk_flops + 2 * 2.0 * Q * N * D, scored_per_s=2 * Q * N / ms * 1e3)
    # one training step (adam, B=128, label smoothing 0.1, dense label rows from the host as the reference's
    # generator ships them, generator.py:160-236)
    from pykg2vec_b200.trainer import Trainer
    cfg = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=0.0001, batch_size=B, neg_rate=0,
                                tot_entity=N, tot_relation=R, label_smoothing=0.1,
                                knowledge_graph=types.SimpleNamespace(read_cache_data=lambda key: {}))
    torch.manual_seed(0)
    np.random.seed(0)
    tmodel = import_model("interacte")(**kw)
    tr = Trainer(tmodel, cfg)
    tr.build_model()
    brng = np.random.RandomState(2)
    Nk = N
    bh, br, bt = brng.randint(Nk, size=B), brng.randint(R, size=B), brng.randint(Nk, size=B)
    lt, lh = np.zeros((B, Nk), np.float32), np.zeros((B, Nk), np.float32)
    lt[np.arange(B), bt] = 1.0
    lh[np.arange(B), bh] = 1.0
    batch = [bh, br, bt, torch.from_numpy(lt), torch.from_numpy(lh)]
    ms = time_ms(lambda: tr.train_batch(batch), args.reps, flush)
    step_flops = 3 * 2 * (2.0 * B * F * D + 2.0 * KS * KS * B * F + 2.0 * B * Nk * D)   # (fwd + 2x fwd for bwd) x 2 dirs
    emit(kernel="InteractE Trainer.train_batch (adam, host dense labels)", case="train B=%d N=%d" % (B, Nk), ms=ms,
         flops=step_flops, h2d_bytes=tr.last_h2d_bytes)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
