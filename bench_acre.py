#!/usr/bin/env python
"""AcrE timings (NOT bench.py, which times the flagship workload) on the FB15k-237 shape (N=14,541, R=237,
hidden_size 200), CUDA events, L2 flushed before every repetition.  Two configurations: the serial way of
hyperparams/AcrE.yaml (in_channels 32, atrous 1/2/2, conv bias) and the CLI default (parallel, in_channels 9,
atrous 1/2/2, conv bias).  One JSON line per measurement, each carrying the card's name and power limit read in
the same run (nvidia-smi --query-gpu, read only):

  trunk        kge_acre_trunk_fwd against the reference's torch layers on the same device (cuDNN dilated convs
               with TF32 off, cuBLAS Linear layers), Q = 512, tail and head direction (AcrE runs the same function
               on (h, r) and (t, r)); every kernel of the trunk is also timed on its own (torch.profiler device
               time, L2 warm)
  rank e2e     Evaluator.rank_triples for 512 filtered queries (serial configuration): host ids in, host ranks out
  train step   one Trainer.train_batch at B = 128 (serial configuration, adam, label smoothing 0.1, host dense
               label rows)

  flops        algorithmic fp32 FLOPs from the shapes, per query: serial convs 2*9*400*(C + 2*C^2), parallel convs
               2*9*400*3*C and gate 2*C*1600*400, fc 2*C*400*200.
Before timing, the script checks that both trunk paths give the same ranks (kernel trunk vs torch layers,
through the same kge_proj_rank): equal, except that a query may differ by the candidates whose prediction is
within the two paths' largest prediction difference of its target's (the trunks round differently; the check
line reports how many queries are equal).  Inputs are fixed-seed.

    python bench_acre.py [--reps 20] [--out results/acre.jsonl]
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

N, R, Q, B, D = 14541, 237, 512, 128, 200
CONFIGS = [("serial", 32, (1, 2, 2)), ("parallel", 9, (1, 2, 2))]
STAGES = ("acre_serial_feature_kernel", "acre_gate_input_kernel", "proj_gemm_kernel", "acre_bn1_relu_kernel",
          "hyper_fc_combine_kernel")


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


def flops(way, C, q):
    conv = 2.0 * 9 * 400 * (C + 2 * C * C) if way == "serial" else 2.0 * 9 * 400 * 3 * C
    gate = 0.0 if way == "serial" else 2.0 * C * 1600 * 400
    return q * conv, q * gate, q * 2.0 * C * 400 * D


def kwargs(way, C, atrous):
    return dict(tot_entity=N, tot_relation=R, hidden_size=D, input_dropout=0.2, hidden_dropout=0.3,
                feature_map_dropout=0.2, in_channels=C, way=way, first_atrous=atrous[0], second_atrous=atrous[1],
                third_atrous=atrous[2], acre_bias=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_acre.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    name, power = card()
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
    serial_model = None
    for way, C, atrous in CONFIGS:
        cfg = "%s C=%d atrous=%d/%d/%d" % (way, C, *atrous)
        torch.manual_seed(0)
        model = import_model("acre")(**kwargs(way, C, atrous))
        with torch.no_grad():   # non-trivial BatchNorm statistics and bias, as a trained model has
            for bn in (model.bn0, model.bn1, model.bn2):
                bn.running_mean.normal_(0.0, 0.2)
                bn.running_var.uniform_(0.5, 1.5)
            model.bias.normal_(0.0, 0.3)
        model = model.to(dev).eval()
        if way == "serial":
            serial_model = model
        ent, bias = (x.detach() for x in model.proj_tail_tables())
        conv_f, gate_f, fc_f = flops(way, C, Q)
        trunk_f = conv_f + gate_f + fc_f
        ws = torch.empty(_lib.acre_trunk_workspace_bytes(way, C, atrous, D, 2 * R, Q), dtype=torch.uint8, device=dev)
        with torch.no_grad():
            # both trunk paths rank alike (same tail kernel, exact counts) before anything is timed.  The two
            # trunks round differently, so a query may only differ by candidates whose prediction lies within the
            # largest prediction difference of the two paths from its target's
            for direction, e, tgt in (("tail", h, t), ("head", t, h)):
                xk = _lib.acre_trunk_fwd(model, e, r, workspace=ws)
                xt = model._trunk_layers(e, r).contiguous()
                ck = _lib.proj_rank(xk, ent, bias, tgt)[:, 0]
                ct = _lib.proj_rank(xt, ent, bias, tgt)[:, 0]
                pk, pt = _lib.proj_tail_fwd(xk, ent, bias), _lib.proj_tail_fwd(xt, ent, bias)
                band = 2 * (pk - pt).abs().max(1, keepdim=True).values
                near = ((pk - pk.gather(1, tgt[:, None])).abs() <= band).sum(1) - 1
                if ((ck - ct).abs() > near).any():
                    raise SystemExit("kernel and torch-layer trunks rank %s queries differently beyond near ties"
                                     % direction)
                emit(check="ranks of kernel trunk vs torch layers", config=cfg, direction=direction, queries=Q,
                     equal=int((ck == ct).sum()), differ_within_near_ties=int((ck != ct).sum()),
                     max_abs_x_diff=float((xk - xt).abs().max()))
            for direction, e in (("tail", h), ("head", t)):
                ms = time_ms(lambda: _lib.acre_trunk_fwd(model, e, r, workspace=ws), args.reps, flush)
                emit(kernel="kge_acre_trunk_fwd", config=cfg, case="eval Q=%d" % Q, direction=direction, ms=ms,
                     flops=trunk_f)
                ms = time_ms(lambda: model._trunk_layers(e, r), args.reps, flush)
                emit(kernel="torch trunk (reference layers: cuDNN convs, cuBLAS Linear)", config=cfg,
                     case="eval Q=%d" % Q, direction=direction, ms=ms, flops=trunk_f)
            # the split: the whole trunk profiled, device time per kernel
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    _lib.acre_trunk_fwd(model, h, r, workspace=ws)
                torch.cuda.synchronize()
            split = {}
            for ev_ in prof.key_averages():
                for tag in STAGES:
                    if tag in ev_.key:
                        split[tag] = split.get(tag, 0.0) + getattr(ev_, "device_time_total", 0.0) / 1e3 / args.reps
            stage_flops = {"acre_serial_feature_kernel": conv_f, "acre_gate_input_kernel": conv_f,
                           "proj_gemm_kernel": gate_f + fc_f}
            for tag in STAGES:
                if tag in split:
                    kw = dict(kernel=tag, config=cfg, case="eval Q=%d, profiled, L2 warm" % Q, ms=split[tag])
                    if stage_flops.get(tag):
                        kw["flops"] = stage_flops[tag]
                    emit(**kw)
            # the reference's layers split the same way
            with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
                for _ in range(args.reps):
                    model._trunk_layers(h, r)
                torch.cuda.synchronize()
            top = sorted(prof.key_averages(), key=lambda ev_: -getattr(ev_, "device_time_total", 0.0))[:6]
            emit(kernel="torch trunk split (top device kernels)", config=cfg, case="eval Q=%d, profiled, L2 warm" % Q,
                 split_ms={ev_.key[:80]: getattr(ev_, "device_time_total", 0.0) / 1e3 / args.reps for ev_ in top})
    with torch.no_grad():
        # end to end: Evaluator.rank_triples on host ids with filters (H2D + trunk x2 + rank x2 + D2H)
        from pykg2vec_b200.evaluator import Evaluator
        ev = object.__new__(Evaluator)
        ev.model, ev.config = serial_model, types.SimpleNamespace(device="cuda", tot_entity=N)
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
        trunk_f = sum(flops("serial", 32, Q))
        emit(kernel="Evaluator.rank_triples AcrE e2e, filtered (host ids in, ranks out)", config="serial C=32",
             case="eval Q=%d" % Q, ms=ms, flops=2 * trunk_f + 2 * 2.0 * Q * N * D, scored_per_s=2 * Q * N / ms * 1e3)
    # one training step (adam, B=128, label smoothing 0.1, dense label rows from the host as the reference's
    # generator ships them, generator.py:160-236)
    from pykg2vec_b200.trainer import Trainer
    cfgns = types.SimpleNamespace(device="cuda", optimizer="adam", learning_rate=0.0001, batch_size=B, neg_rate=0,
                                  tot_entity=N, tot_relation=R, label_smoothing=0.1,
                                  knowledge_graph=types.SimpleNamespace(read_cache_data=lambda key: {}))
    torch.manual_seed(0)
    tmodel = import_model("acre")(**kwargs("serial", 32, (1, 2, 2)))
    tr = Trainer(tmodel, cfgns)
    tr.build_model()
    brng = np.random.RandomState(2)
    bh, br, bt = brng.randint(N, size=B), brng.randint(R, size=B), brng.randint(N, size=B)
    lt, lh = np.zeros((B, N), np.float32), np.zeros((B, N), np.float32)
    lt[np.arange(B), bt] = 1.0
    lh[np.arange(B), bh] = 1.0
    batch = [bh, br, bt, torch.from_numpy(lt), torch.from_numpy(lh)]
    ms = time_ms(lambda: tr.train_batch(batch), args.reps, flush)
    step_flops = 3 * 2 * (sum(flops("serial", 32, B)) + 2.0 * B * N * D)   # (fwd + 2x fwd for bwd) x 2 dirs
    emit(kernel="AcrE Trainer.train_batch (adam, host dense labels)", config="serial C=32",
         case="train B=%d N=%d" % (B, N), ms=ms, flops=step_flops, h2d_bytes=tr.last_h2d_bytes)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            for line in lines:
                f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
