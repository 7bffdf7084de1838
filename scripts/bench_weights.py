"""Device time of a weighted train step against an unweighted one, on bench.py's configurations.

    python scripts/bench_weights.py [--steps 200] [--warmup 20] [--workloads fm_c2,ffm_c3,nfm_c4]

  fm_c2   FM k=16, batch 4096 (C2)    ffm_c3  FFM k=4, 39 fields, batch 8192, FTRL (C3)
  nfm_c4  NFM k=16 + [256, 128, 64] on the tensor cores (bf16), batch 16384 (C4)

Two contexts of the workload on the same resident batches, one of them with per-row weights in [0, 4) on every slot.
Their steps alternate in one loop, each bracketed by CUDA events on its context's stream after an L2 flush (256 MB
zeroed, as bench.py does), after `warmup` steps of each.  Reports the median step of each and their difference; the
card's name, power limit and max SM clock are read in the same run.  One JSON line per workload."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--workloads", default="fm_c2,ffm_c3,nfm_c4")
    args = ap.parse_args()
    import torch
    from lightctr_b200 import build
    build.build()
    if not torch.cuda.is_available():
        raise SystemExit("bench_weights.py: no CUDA device")
    c = card()
    for name in args.workloads.split(","):
        print(json.dumps(dict(measure(name, args.steps, args.warmup), **c)), flush=True)


if __name__ == "__main__":
    main()
