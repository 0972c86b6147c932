"""Batched top-k link prediction (Evaluator.predict_tails / predict_heads) at the FB15k-237 shape: N = 14,541,
R = 237, d = 200, for TransE-L2, DistMult, ComplEx, RotatE, TransH and ConvE (hidden_size_1 = 20); Q in
{1, 512, 20,466}, k in {10, 100}, raw and filtered (known positives of a dataset-shaped synthetic graph).

One JSON line per measurement, each carrying the card's name and power limit read in the same run
(nvidia-smi --query-gpu, read only):
  * ms                  wall clock of predict_tails, host ids in -> host ids / scores out (it ends in a device sync),
                        median of the timed calls after one warm-up call;
  * producer_share / select_share   device time of the score producer (topk_store_kernel, or the tail GEMM and the
                        trunk for ConvE) and of topk_select_kernel over all device time of one call, from a separate
                        torch.profiler run;
  * torch_ms            the same work done with torch: model.forward over expanded ids in chunks of 64 queries,
                        masked_fill for the filter, torch.topk;
  * per_query_ms        today's route, Evaluator.test_tail_rank(h, r, topk=k) once per query (raw only; timed over the
                        first min(Q, 512) queries and reported per query).
The script asserts that predict_tails' ids equal the torch route's on every query whose torch top-(k+1) scores are
separated by more than 1e-5 relative (tie-free), and reports how many queries that was.

    python bench_topk.py [--models transe,conve] [--out results.jsonl]
"""
import argparse
import json
import subprocess
import time

import numpy as np
import torch

N, R, D, QTEST = 14541, 237, 200, 20466
QS, KS = (1, 512, QTEST), (10, 100)
MODELS = {
    "transe": dict(l1_flag=False), "distmult": {}, "complex": {}, "rotate": dict(margin=6.0), "transh": dict(l1_flag=False),
    "conve": dict(hidden_size_1=20, input_dropout=0.0, feature_map_dropout=0.0, hidden_dropout=0.0, lmbda=0.1),
}
PRODUCER = ("topk_store_kernel", "proj_gemm_kernel", "conve")
CHUNK = 64


def card():
    """(name, power limit) of GPU 0 as nvidia-smi reports them: the limit in W, or nvidia-smi's own text when it
    gives no number (e.g. "[N/A]")"""
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


def wall_ms(fn, reps):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(out))


def shares(fn):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    total = prod = sel = 0.0
    for e in prof.events():   # device-side kernel records only (CPU ops would count their kernels twice)
        if e.device_type != DeviceType.CUDA or e.name.startswith("Memcpy") or e.name.startswith("Memset"):
            continue
        t = e.time_range.elapsed_us()
        total += t
        if "topk_select_kernel" in e.name:
            sel += t
        elif any(p in e.name for p in PRODUCER):
            prod += t
    return (prod / total if total else None), (sel / total if total else None)


def torch_route(model, proj, hs, rs, k, filt, dev):
    """chunked model.forward + masked_fill + torch.topk -> (ids [Q,k], scores [Q,k]) of the best first"""
    ids, scores = [], []
    ent = torch.arange(N, device=dev)
    with torch.no_grad():
        for lo in range(0, len(hs), CHUNK):
            hi = min(len(hs), lo + CHUNK)
            c = hi - lo
            h = torch.from_numpy(hs[lo:hi]).to(dev)
            r = torch.from_numpy(rs[lo:hi]).to(dev)
            if proj:
                s = model.forward(h, r, direction="tail")
            else:
                s = model.forward(h.repeat_interleave(N), r.repeat_interleave(N), ent.repeat(c)).view(c, N)
            if filt is not None:
                ptr, idx = filt
                lens = torch.from_numpy(np.diff(ptr[lo:hi + 1])).to(dev)
                rows = torch.repeat_interleave(torch.arange(c, device=dev), lens)
                mask = torch.zeros((c, N), dtype=torch.bool, device=dev)
                mask[rows, torch.from_numpy(idx[ptr[lo]:ptr[hi]]).to(dev)] = True
                s = s.masked_fill(mask, float("-inf") if proj else float("inf"))
            v, i = torch.topk(s, k, dim=1, largest=proj)
            ids.append(i)
            scores.append(v)
    return torch.cat(ids).cpu().numpy(), torch.cat(scores).cpu().numpy()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--models", default=",".join(MODELS))
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_topk.py needs a CUDA device")
    import pykg2vec_b200
    from pykg2vec_b200.evaluator import Evaluator, build_filter_csr
    from pykg2vec_b200.synthetic import SyntheticConfig, SyntheticKnowledgeGraph
    dev = torch.device("cuda", 0)
    name, power = card()
    kg = SyntheticKnowledgeGraph.shaped_like("fb15k_237", seed=0)
    test = kg.arrays["test"]

    def emit(**kw):
        kw.update(gpu=name, power_limit_w=power)
        print(json.dumps(kw), flush=True)
        if args.out:
            with open(args.out, "a") as f:
                f.write(json.dumps(kw) + "\n")

    for mname in args.models.split(","):
        cfg = SyntheticConfig(kg, device="cuda", hidden_size=D, **MODELS[mname])
        torch.manual_seed(0)
        model = pykg2vec_b200.import_model(mname)(**cfg.__dict__).cuda().eval()
        ev = Evaluator(model, cfg)
        proj = hasattr(model, "proj_query")
        for Q in QS:
            hs, rs = test[:Q, 0].copy(), test[:Q, 1].copy()
            filt = build_filter_csr(list(zip(hs.tolist(), rs.tolist())), ev.metric_calculator.hr_t)
            for k in KS:
                for filtered in (False, True):
                    reps = 20 if Q == 1 else (5 if Q == 512 else 3)
                    call = lambda: ev.predict_tails(hs, rs, k=k, filtered=filtered)
                    ms = wall_ms(call, reps)
                    prod, sel = shares(call)
                    ids, sc = call()
                    f = filt if filtered else None
                    t_ms = wall_ms(lambda: torch_route(model, proj, hs, rs, k, f, dev), 1 if Q == QTEST else 3)
                    t_ids, t_sc = torch_route(model, proj, hs, rs, k + 1 if k < 256 else k, f, dev)
                    gaps = np.abs(np.diff(t_sc.astype(np.float64), axis=1)) > 1e-5 * np.maximum(
                        np.abs(t_sc[:, 1:]).astype(np.float64), 1e-30)
                    clean = np.all(gaps, axis=1) & np.all(np.isfinite(t_sc), axis=1)
                    assert np.array_equal(ids[clean], t_ids[clean, :k]), (mname, Q, k, filtered)
                    row = dict(model=mname, N=N, d=D, Q=Q, k=k, filtered=filtered, ms=ms, ms_per_query=ms / Q,
                               producer_share=prod, select_share=sel, torch_ms=t_ms,
                               torch_checked_queries=int(clean.sum()))
                    if not filtered:
                        nq = min(Q, 512)
                        with torch.no_grad():
                            pq = wall_ms(lambda: [ev.test_tail_rank(int(hs[i]), int(rs[i]), topk=k) for i in range(nq)],
                                         1)
                        row.update(per_query_ms=pq / nq, per_query_queries_timed=nq)
                    emit(**row)
        del model, ev
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
