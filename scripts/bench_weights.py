"""Device time of a weighted train step against an unweighted one, on bench.py's configurations.

    python scripts/bench_weights.py [--steps 200] [--warmup 20] [--workloads fm_c2,ffm_c3,nfm_c4]
    python scripts/bench_weights.py --stream [--steps 400] [--blocks 6] [--workloads fm_c2,nfm_c4]
    python scripts/bench_weights.py --eval [--rows 1048576,16777216]

  fm_c2   FM k=16, batch 4096 (C2)    ffm_c3  FFM k=4, 39 fields, batch 8192, FTRL (C3)
  nfm_c4  NFM k=16 + [256, 128, 64] on the tensor cores (bf16), batch 16384 (C4)

Two contexts of the workload on the same resident batches, one of them with per-row weights in [0, 4) on every slot.
Their steps alternate in one loop, each bracketed by CUDA events on its context's stream after an L2 flush (256 MB
zeroed, as bench.py does), after `warmup` steps of each.  Reports the median step of each and their difference; the
card's name, power limit and max SM clock are read in the same run.  One JSON line per workload.

--stream: end-to-end samples/s of the streamed pipeline (bench.py's end-to-end arm: pinned host batches in, statistics out
every step, LCTR_PIPE_DEPTH in flight), weighted (lctr_train_batch_weighted_async, pinned weights in [0, 4)) against
unweighted (lctr_train_batch_async) on one context, alternated in blocks of `steps` steps, each block after a synchronise.
Reports the median block of each kind.

--eval: host time of lctr_eval_pred_weighted against lctr_eval_pred on n random (pCTR, label, weight) rows, each call
synchronous (copies in, kernels, three numbers out), alternated, median of `steps` calls after `warmup` at 1 M rows and
proportionally fewer (at least 3, after one warm-up) at more rows: the one-warp chains take time linear in n."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

import numpy as np  # noqa: E402

from bench import N_FIELDS, WORKLOADS, make_batches  # noqa: E402
from bench_score import card, make_context  # noqa: E402


def measure(name, steps, warmup):
    import torch
    from lightctr_b200 import capi
    wl = dict(WORKLOADS[name])
    B = wl["batch"]
    nb = wl.get("nb", 8)
    batches = make_batches(wl, nb)
    ctxs = [make_context(capi, wl, B) for _ in range(2)]
    rng = np.random.default_rng(5)
    for ctx in ctxs:
        for i, (rp, fid, fld, lab) in enumerate(batches):
            ctx.upload_batch(i, rp, fid, fld if wl["model"] == "ffm" else None, None, lab)
    for i in range(nb):
        ctxs[1].set_row_weights(i, (rng.random(B) * 4).astype(np.float32))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    streams = [torch.cuda.ExternalStream(c.stream()) for c in ctxs]
    times = [[], []]
    for it in range(warmup + steps):
        for j, (ctx, st) in enumerate(zip(ctxs, streams)):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(st):
                flush.zero_()
                a.record(st)
            ctx.train_step(it % nb, want_stats=False)
            with torch.cuda.stream(st):
                b.record(st)
            b.synchronize()
            if it >= warmup:
                times[j].append(a.elapsed_time(b) * 1e3)
    for ctx in ctxs:
        ctx.close()
    plain, weighted = (float(np.median(t)) for t in times)
    return dict(workload=name, rows=B, steps=steps, unweighted_us=plain, weighted_us=weighted, delta_us=weighted - plain,
                delta_pct=100.0 * (weighted - plain) / plain)


def _pinned(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).pin_memory().numpy()


def measure_stream(name, steps, blocks):
    import time
    from lightctr_b200 import capi
    wl = dict(WORKLOADS[name])
    B = wl["batch"]
    nb = wl.get("nb", 8)
    Fc = N_FIELDS if wl["model"] == "ffm" else 0
    host = [(_pinned(rp), _pinned(fid), _pinned(fld) if Fc else None, None, _pinned(lab))
            for rp, fid, fld, lab in make_batches(wl, nb)]
    rng = np.random.default_rng(5)
    weights = [_pinned((rng.random(B) * 4).astype(np.float32)) for _ in range(nb)]
    ctx = make_context(capi, wl, B)

    def run(n, weighted):
        pending = []
        for i in range(n):
            kw = {"weight": weights[i % nb]} if weighted else {}
            pending.append(ctx.train_batch_async(*host[i % nb], **kw))
            if len(pending) >= capi.PIPE_DEPTH:
                ctx.wait(pending.pop(0))
        for t in pending:
            ctx.wait(t)
        ctx.sync()

    for weighted in (False, True):  # warm-up: both kinds through every pipeline slot
        run(nb + 3, weighted)
    rates = [[], []]
    for blk in range(2 * blocks):
        weighted = blk % 2 == 1
        t0 = time.perf_counter()
        run(steps, weighted)
        rates[weighted].append(B * steps / (time.perf_counter() - t0))
    ctx.close()
    plain, weighted = (float(np.median(r)) for r in rates)
    return dict(arm="stream", workload=name, rows=B, steps_per_block=steps, blocks=blocks, unweighted_samples_s=plain,
                weighted_samples_s=weighted, delta_pct=100.0 * (weighted - plain) / plain)


def measure_eval(n, steps, warmup):
    import time
    from lightctr_b200 import capi
    rng = np.random.default_rng(7)
    p = rng.random(n).astype(np.float32)
    y = (rng.random(n) < 0.25).astype(np.int32)
    w = (rng.random(n) * 4).astype(np.float32)
    ctx = capi.Context(capi.MODEL_FM, 1000, 8)
    if n > (1 << 20):
        steps, warmup = max(3, steps * (1 << 20) // n), 1
    times = [[], []]
    for it in range(warmup + steps):
        for j in range(2):
            t0 = time.perf_counter()
            ctx.eval_pred(p, y, w if j else None)
            if it >= warmup:
                times[j].append((time.perf_counter() - t0) * 1e3)
    ctx.close()
    plain, weighted = (float(np.median(t)) for t in times)
    return dict(arm="eval", rows=n, calls=steps, eval_pred_ms=plain, eval_pred_weighted_ms=weighted,
                ratio=weighted / plain)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--workloads", default=None)
    ap.add_argument("--stream", action="store_true")
    ap.add_argument("--blocks", type=int, default=6)
    ap.add_argument("--eval", action="store_true")
    ap.add_argument("--rows", default="1048576,16777216")
    args = ap.parse_args()
    import torch
    from lightctr_b200 import build
    build.build()
    if not torch.cuda.is_available():
        raise SystemExit("bench_weights.py: no CUDA device")
    c = card()
    if args.stream:
        for name in (args.workloads or "fm_c2,nfm_c4").split(","):
            print(json.dumps(dict(measure_stream(name, args.steps, args.blocks), **c)), flush=True)
    if args.eval:
        for n in args.rows.split(","):
            print(json.dumps(dict(measure_eval(int(n), args.steps, args.warmup), **c)), flush=True)
    if not (args.stream or args.eval):
        for name in (args.workloads or "fm_c2,ffm_c3,nfm_c4").split(","):
            print(json.dumps(dict(measure(name, args.steps, args.warmup), **c)), flush=True)


if __name__ == "__main__":
    main()
