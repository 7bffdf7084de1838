"""Device time of lctr_score against lctr_train_step on the same batch, on bench.py's configurations.

    python scripts/bench_score.py [--calls 200] [--warmup 20] [--workloads nfm_c4,nfm_c4_1m,fm_c2,ffm_c3]

  nfm_c4     NFM k=16 + [256, 128, 64] on the tensor cores (bf16), batch 16384 (bench.py's C4)
  nfm_c4_1m  the same context scoring a 1,048,576-row slot whole (16 blocks of 65536 rows); no step at that size
  fm_c2      FM k=16, batch 4096 (C2)          ffm_c3  FFM k=4, 39 fields, batch 8192, FTRL (C3)

Per workload: the median of `calls` timed calls of each kind, score and step alternated in the same loop, each bracketed
by CUDA events on the context's stream (lctr_stream) after `warmup` calls of each; rows per second of a score; and, in a
run of its own with lctr_profile on, the share of the dense layers (PROF_MLP) in the profiled time of a score and of a
step.  The card's name, power limit and max SM clock are read in the same run.  One JSON line per workload."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import N_FIELDS, WORKLOADS, make_batches  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True, check=True)
    name, power, clock = (s.strip() for s in q.stdout.strip().split("\n")[0].split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def make_context(capi, wl, B):
    """bench.py's context of the workload (synthetic parameters on the device; C4's chain U(-0.5, 0.5), bias 0)"""
    model = {"fm": capi.MODEL_FM, "ffm": capi.MODEL_FFM, "nfm": capi.MODEL_NFM}[wl["model"]]
    opt = {"adagrad": capi.OPT_ADAGRAD, "ftrl": capi.OPT_FTRL}[wl["opt"]]
    k = wl["k"]
    ctx = capi.Context(model, wl["F"], k, N_FIELDS if wl["model"] == "ffm" else 0, optimizer=opt, max_nnz=B * 100,
                       hidden=wl.get("hidden", ()), mlp_precision=capi.MLP_BF16 if wl["model"] == "nfm" else capi.MLP_FP32)
    if wl["model"] == "nfm":
        rng = np.random.default_rng(99)
        dims = [k] + list(wl["hidden"]) + [1]
        for li in range(len(dims) - 1):
            ctx.mlp_upload(li, rng.random((dims[li + 1], dims[li]), dtype=np.float32) - 0.5, np.zeros(dims[li + 1], np.float32))
    ctx.fill_params(1234, float(1.0 / np.sqrt(k)))
    return ctx


def upload(ctx, wl, slot, batches):
    rp = [np.zeros(1, np.int64)]
    off = 0
    for b in batches:
        rp.append(b[0][1:] + off)
        off += int(b[0][-1])
    rp, fid, fld, lab = (np.concatenate(rp),) + tuple(np.concatenate([b[i] for b in batches]) for i in (1, 2, 3))
    ctx.upload_batch(slot, rp, fid, fld if wl["model"] == "ffm" else None, None, lab)
    return len(rp) - 1


def median_times(torch, ctx, fns, calls, warmup):
    """{name: median ms} of the callables in fns, called in turn (alternated), each bracketed by events on lctr_stream"""
    st = torch.cuda.ExternalStream(ctx.stream())
    for _ in range(warmup):
        for fn in fns.values():
            fn()
    ctx.sync()
    ts = {name: [] for name in fns}
    for _ in range(calls):
        for name, fn in fns.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(st)
            fn()
            b.record(st)
            b.synchronize()
            ts[name].append(a.elapsed_time(b))
    return {name: float(np.median(v)) for name, v in ts.items()}


def dense_share(ctx, fn, n):
    ctx.sync()
    ctx.profile_read(reset=True)
    ctx.profile(True)
    for _ in range(n):
        fn()
    prof = ctx.profile_read(reset=True)
    ctx.profile(False)
    total = sum(ms for ms, _ in prof.values())
    return (prof.get("mlp", (0.0, 0))[0] / total) if total else None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--workloads", default="nfm_c4,nfm_c4_1m,fm_c2,ffm_c3")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_score: no GPU (a timing needs one)")
    from lightctr_b200 import build as lbuild
    lbuild.build()
    from lightctr_b200 import capi
    info = card()
    for name in args.workloads.split(","):
        big = name == "nfm_c4_1m"
        wl = dict(WORKLOADS["nfm_c4" if big else name])
        B = wl["batch"]
        ctx = make_context(capi, wl, B)
        rows = upload(ctx, wl, 0, make_batches(wl, 1))
        res = dict(workload=name, desc=wl["desc"] + ("; 1,048,576-row slot scored whole" if big else ""), rows=rows, **info)
        if big:
            n = (1 << 20) // B
            rows = upload(ctx, wl, 1, make_batches(wl, n, seed_offset=1))
            calls = max(5, args.calls // 20)
            t = median_times(torch, ctx, {"score": lambda: ctx.score(1, download=False)}, calls, 2)
            res.update(rows=rows, calls=calls, score_ms=t["score"], score_rows_per_s=rows / t["score"] * 1e3,
                       score_dense_share=dense_share(ctx, lambda: ctx.score(1, download=False), 3))
        else:
            t = median_times(torch, ctx, {"score": lambda: ctx.score(0, download=False),
                                          "step": lambda: ctx.train_step(0, want_stats=False)}, args.calls, args.warmup)
            res.update(calls=args.calls, score_ms=t["score"], step_ms=t["step"], score_over_step=t["score"] / t["step"],
                       score_rows_per_s=rows / t["score"] * 1e3,
                       score_dense_share=dense_share(ctx, lambda: ctx.score(0, download=False), 20),
                       step_dense_share=dense_share(ctx, lambda: ctx.train_step(0, want_stats=False), 20))
        ctx.close()
        print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
