"""measurement aid: per-kernel CUDA time of bench.py's resident step, from torch.profiler

    python profiles/step_breakdown.py [--reps 30] [--out FILE.json]

Builds the bench workload with bench.py's own make_graph / build / make_batches, captures the three CUDA
graphs bench.py times (the whole single-GPU step, its training half, its evaluation half) the same way, and
replays each `--reps` times under torch.profiler with the L2 flushed (256 MiB memset, as bench.py does) before
every replay.  Prints one JSON object: per graph, every device activity (kernels and memsets) by name with its
launches per replay and mean microseconds per replay, the sum of those, and the CUDA-event time of one replay
taken without the profiler.  The flush's own kernel is left out of the tables.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from pykg2vec_b200 import _lib  # noqa: E402


def device_events(prof):
    cuda = torch.autograd.DeviceType.CUDA
    return [e for e in prof.events() if e.device_type == cuda]


def profile(fn, flush, reps):
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            flush.zero_()
            torch.cuda.synchronize()
            fn()
            torch.cuda.synchronize()
    return device_events(prof)


def event_us(fn, flush, reps):
    tot = 0.0
    for _ in range(reps):
        flush.zero_()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        tot += a.elapsed_time(b)
    return tot * 1e3 / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=30)
    ap.add_argument("--out", default=None, help="also write the JSON object to this file")
    args = ap.parse_args()
    w = bench.WORKLOAD
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    kg = bench.make_graph()
    tr = bench.build(kg, dev)
    (ids, q), = bench.make_batches(kg, 1, 0)
    from pykg2vec_b200.evaluator import build_filter_csr
    hr_t, tr_h = kg.read_cache_data("hr_t"), kg.read_cache_data("tr_h")
    ft = build_filter_csr([(int(h), int(r)) for h, r, t in q], hr_t)
    fh = build_filter_csr([(int(t), int(r)) for h, r, t in q], tr_h)
    tod = lambda a: torch.from_numpy(a.astype("int64")).to(dev)   # noqa: E731
    s_ids = [tod(a) for a in ids]
    qh, qr, qt = tod(q[:, 0]), tod(q[:, 1]), tod(q[:, 2])
    ft, fh = (tod(ft[0]), tod(ft[1])), (tod(fh[0]), tod(fh[1]))
    desc = tr.model.kge_desc()
    counts = torch.zeros((w["Q"], 4), dtype=torch.int32, device=dev)
    ws = torch.empty(max(_lib.rank_workspace_bytes(desc, w["Q"]), 16), dtype=torch.uint8, device=dev)
    flush = torch.empty(bench.L2_FLUSH_BYTES, dtype=torch.uint8, device=dev)
    scratch = tr._grad_scratch
    loss_buf = torch.zeros(1, dtype=torch.float32, device=dev)

    def body_eval():
        counts.zero_()
        _lib.rank_1vsall(desc, qh, qr, qt, ft, fh, counts=counts, workspace=ws)

    def body_train(lr):
        _lib.train_pairwise_hinge_sgd(desc, scratch, *s_ids, w["margin"], lr, loss_buf)

    def body_step(lr):
        body_eval()
        body_train(lr)

    def capture(fn, warm):   # as bench.py captures: un-captured warm-up on a side stream, then one capture
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            warm()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            fn()
        return g

    # lr = 0 everywhere: replays leave the tables as they are, so every replay does the same work
    graphs = {"step": capture(lambda: body_step(0.0), lambda: body_step(0.0)),
              "train": capture(lambda: body_train(0.0), lambda: body_train(0.0)),
              "eval": capture(body_eval, body_eval)}
    for g in graphs.values():
        for _ in range(5):
            g.replay()
    torch.cuda.synchronize()
    flush_names = {e.name for e in profile(lambda: None, flush, 3)}
    props = torch.cuda.get_device_properties(dev)
    out = {"gpu": props.name, "reps": args.reps, "l2_flushed_before_every_replay": True, "graphs": {}}
    try:
        import subprocess
        out["power_limit_w"] = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                                              capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:   # noqa: BLE001 — informational only
        out["power_limit_w"] = None
    for name, g in graphs.items():
        evs = [e for e in profile(g.replay, flush, args.reps) if e.name not in flush_names]
        per = {}
        for e in evs:
            k = per.setdefault(e.name, [0, 0.0])
            k[0] += 1
            k[1] += e.time_range.elapsed_us()
        rows = sorted(({"name": n, "launches_per_replay": c / args.reps, "us_per_replay": t / args.reps}
                       for n, (c, t) in per.items()), key=lambda r: -r["us_per_replay"])
        out["graphs"][name] = {"kernels": rows, "sum_us": sum(r["us_per_replay"] for r in rows),
                               "replay_event_us": event_us(g.replay, flush, args.reps)}
    step = out["graphs"]["step"]["kernels"]
    out["train_in_step_us"] = sum(r["us_per_replay"] for r in step
                                  if "train_hinge_kernel" in r["name"] or "apply_rows_kernel" in r["name"]
                                  or r["name"].startswith("Memset"))
    text = json.dumps(out, indent=1)
    print(text)
    if args.out:
        with open(args.out, "w") as f:
            f.write(text)


if __name__ == "__main__":
    main()
