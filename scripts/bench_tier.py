#!/usr/bin/env python
"""Host tier of a keyed context (cfg.key_host_rows) on one GPU, on the C2 shape: FM k = 16, Adagrad, device capacity 1M
rows, batches of 4096 rows x 39 keys.  Tiered (key_host_rows = 500K) and untiered (key_evict = 1) contexts are alternated
in one process, --rounds times.

    python scripts/bench_tier.py [--rounds R] [--steps K]

Both contexts start each measurement from the same full table of 1M rows whose ages are spread uniformly over 0..99
(seeded with lctr_upload_keyed_params between empty insert-uploads, then restored from a checkpoint in a temporary
directory).  Prints ONE JSON line:
  evict_ms            host clock around lctr_evict_keys (it ends in a stream synchronise) freeing 10 / 25 / 50 % of the
                      rows through max_rows, tiered (rows spilled into pinned host memory) and untiered (rows dropped);
  evict_tier_ms       lctr_evict_host_tier freeing half of a full tier of 500K rows;
  upload_ms           host clock around lctr_upload_batch_keys (insert = 1, ends in a synchronise) of a batch of resident
                      keys with 0, 1 and 10 % of its entries replaced by keys held in the tier, and untiered at 0 %;
  step_ms             train step (host clock over --steps steps ending in a synchronise), tiered and untiered;
  restore_vs_tier_ms  the upload above with 0, 1 and 10 % of its entries restored, on contexts whose tier holds 0.5 M and
                      4 M rows (half and four times the device capacity; the device table half full): the restore and
                      the compaction after it cost in proportion to the rows restored, not to the tier;
  gpu                 card name, power limit and maximum SM clock, read in the same run.
Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only

import numpy as np  # noqa: E402

from lightctr_b200.dist import fmix64  # noqa: E402

CAP, K, ROWS, PER, TIER = 1_000_000, 16, 4096, 39, 500_000


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def upload(ctx, keys, slot=0):
    rp = np.arange(0, len(keys) + 1, PER, dtype=np.int64)
    lab = (fmix64(keys[::PER]) & np.uint64(3) == 0).astype(np.int32)
    ctx.upload_batch_keys(slot, rp, keys, None, None, lab)


def timed(fn):
    t0 = time.perf_counter()
    out = fn()
    return (time.perf_counter() - t0) * 1e3, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=200)
    args = ap.parse_args()
    from lightctr_b200 import capi
    universe = fmix64(np.arange(CAP, dtype=np.uint64) + np.uint64(1 << 48))
    ctxs = {name: capi.Context(capi.MODEL_FM, CAP, K, key_mode=capi.KEYS_HASHED, key_evict=True, key_host_rows=tier)
            for name, tier in (("tiered", TIER), ("untiered", 0))}
    res = {"evict_ms": {}, "evict_tier_ms": [], "upload_ms": {}, "step_ms": {}, "gpu": gpu_info(),
           "shape": "FM k=16 Adagrad, capacity %d rows, tier %d rows, batch %d x %d keys" % (CAP, TIER, ROWS, PER)}
    with tempfile.TemporaryDirectory() as tmp:
        ck = {}
        for name, ctx in ctxs.items():  # 100 chunks of 10K keys, one empty insert-upload between: ages 99 .. 0
            for c in range(100):
                ctx.upload_keyed_params(universe[c * 10000:(c + 1) * 10000])
                ctx.upload_batch_keys(7, np.zeros(1, np.int64), np.zeros(0, np.uint64), None, None, np.zeros(0, np.int32))
            ck[name] = os.path.join(tmp, name + ".ckpt")
            ctx.save_checkpoint(ck[name])
        rng = np.random.default_rng(0)
        for rnd in range(args.rounds):
            for frac in (0.10, 0.25, 0.50):
                for name, ctx in ctxs.items():
                    ctx.load_checkpoint(ck[name])
                    ms, n = timed(lambda: ctx.evict_keys(max_rows=int(CAP * (1 - frac))))
                    res["evict_ms"].setdefault("%s_%d%%" % (name, frac * 100), []).append(round(ms, 3))
            # the tiered context now holds a full tier of 500K rows (the 50 % eviction)
            t, u = ctxs["tiered"], ctxs["untiered"]
            ms, _ = timed(lambda: t.evict_host_tier(max_rows=TIER // 2))
            res["evict_tier_ms"].append(round(ms, 3))
            tier_keys = t.download_host_tier()[0]
            resident = t.download_keys()
            used = 0
            for name, ctx, frac in (("untiered_0%", u, 0.0), ("tiered_0%", t, 0.0), ("tiered_1%", t, 0.01), ("tiered_10%", t, 0.10)):
                src = resident if ctx is t else u.download_keys()
                keys = src[rng.integers(0, len(src), ROWS * PER)]
                m = int(round(len(keys) * frac))
                if m:  # distinct tier keys, each met once
                    keys[rng.choice(len(keys), m, replace=False)] = tier_keys[used:used + m]
                    used += m
                ms, _ = timed(lambda: upload(ctx, keys))
                res["upload_ms"].setdefault(name, []).append(round(ms, 3))
            # step time: the same batch of resident keys on both contexts
            for name, ctx in ctxs.items():
                upload(ctx, ctx.download_keys()[rng.integers(0, CAP // 4, ROWS * PER)], slot=1)
                for _ in range(10):
                    ctx.train_step(1, want_stats=False)
                ctx.sync()
                ms, _ = timed(lambda: ([ctx.train_step(1, want_stats=False) for _ in range(args.steps)], ctx.sync()))
                res["step_ms"].setdefault(name, []).append(round(ms / args.steps, 5))
    for ctx in ctxs.values():
        ctx.close()
    res["restore_vs_tier_ms"] = restore_vs_tier(capi, args.rounds)
    print(json.dumps(res))


def restore_vs_tier(capi, rounds):
    out = {}
    rng = np.random.default_rng(1)
    for size in (TIER, 4 * CAP):
        ctx = capi.Context(capi.MODEL_FM, CAP, K, key_mode=capi.KEYS_HASHED, key_evict=True, key_host_rows=size)
        base = np.uint64(1 << 50)
        for c in range(size // TIER):  # fill the tier 500K rows at a time
            ctx.upload_keyed_params(fmix64(np.arange(c * TIER, (c + 1) * TIER, dtype=np.uint64) + base))
            ctx.evict_keys(max_rows=0)
        ctx.upload_keyed_params(fmix64(np.arange(size, size + CAP // 2, dtype=np.uint64) + base))
        resident, tier_keys = ctx.download_keys(), ctx.download_host_tier()[0]
        rng.shuffle(tier_keys)
        used = 0
        for rnd in range(rounds + 1):  # the first round warms up
            for frac in (0.0, 0.01, 0.10):
                keys = resident[rng.integers(0, len(resident), ROWS * PER)]
                m = int(round(len(keys) * frac))
                if m:
                    keys[rng.choice(len(keys), m, replace=False)] = tier_keys[used:used + m]
                    used += m
                ms, _ = timed(lambda: upload(ctx, keys))
                if rnd:
                    out.setdefault("tier_%dK_%d%%" % (size // 1000, frac * 100), []).append(round(ms, 3))
        ctx.close()
    return out


if __name__ == "__main__":
    main()
