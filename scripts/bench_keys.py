#!/usr/bin/env python
"""Keyed mode against dense mode on one GPU: the same workload and batches, ids fed as 64-bit keys fmix64(fid) into a keyed
context of capacity F (cfg.key_mode = LCTR_KEYS_HASHED), alternated with the dense context in one process.

    python scripts/bench_keys.py [--workload fm_c2|ffm_c3|nfm_c4] [--steps K] [--warmup W] [--rounds R] [--evict | --admit]

Prints ONE JSON line:
  keyed_ms_per_step / dense_ms_per_step   device-timed step (one CUDA-event pair per step, L2 flushed before each step,
                                          as bench.py times `value`), one entry per round;
  translate_us_per_batch                  device time of the upload-side insert + lazy init + translate launches (the
                                          library's per-launch events, L2 not flushed): first upload of each batch
                                          ("first_sight": new keys get rows; "first_batch": the first one, on an empty
                                          table) and a second upload of the same batches ("all_known": probes only);
  table_bytes                             key table (slots of u64 key + u32 row, u64 key per row) and lctr_device_bytes;
  gpu                                     card name and power limit, read in the same run.
With --evict (row eviction, cfg.key_evict; the workload is then always fm_c2: capacity 1M, k = 16, Adagrad) the line
instead holds, per round:
  translate_us_per_batch                  as above for keyed contexts with key_evict = 1 ("tracked", stamps stored by the
                                          translate launch) and 0 ("untracked"), alternated;
  ms_per_step                             step time of the dense, untracked and tracked contexts, alternated;
  evict_ms                                host clock around lctr_evict_keys (it ends in a stream synchronise) on a full
                                          table of 1M rows whose ages are spread uniformly over 0..99, evicting 10 %, 25 %
                                          and 50 % of them through max_rows, with and without export of keys, W and V;
  rows_moved                              survivors renumbered by each of those calls.
With --admit (frequency admission, lctr_set_key_admission; workload fm_c2, capacity 1M, sketch 4 x 2^22) the line holds,
for admission off and at min_count 2 and 4, contexts alternated within each round:
  translate_us_per_batch                  device time of the upload-side key launches (count, admit, init, translate and
                                          the compaction of dropped entries) per batch, over a first and a second pass of
                                          the same batches ("pass1", "pass2");
  upload_ms_per_batch                     host clock around lctr_upload_batch_keys (it ends in a stream synchronise);
  rows_created                            rows held after each pass (exact), and "model": the same counts from a numpy
                                          restatement of the sketch and the admission rule;
  dropped_entries                         entries dropped over each pass.
Writes nothing to the tree (the full table is restored from a checkpoint in a temporary directory).
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

from bench import N_FIELDS, WORKLOADS, make_batches  # noqa: E402
from lightctr_b200.dist import fmix64  # noqa: E402


def gpu_info():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def run(wl, batches, keyed, steps, warmup, key_evict=False):
    import torch
    from lightctr_b200 import capi
    model = {"fm": capi.MODEL_FM, "ffm": capi.MODEL_FFM, "nfm": capi.MODEL_NFM}[wl["model"]]
    opt = {"adagrad": capi.OPT_ADAGRAD, "ftrl": capi.OPT_FTRL}[wl["opt"]]
    F, k, B = wl["F"], wl["k"], wl["batch"]
    Fc = N_FIELDS if wl["model"] == "ffm" else 0
    ctx = capi.Context(model, F, k, Fc, optimizer=opt, max_nnz=B * 100, hidden=wl.get("hidden", ()),
                       mlp_precision=capi.MLP_BF16 if wl["model"] == "nfm" else capi.MLP_FP32,
                       key_mode=capi.KEYS_HASHED if keyed else capi.KEYS_DENSE, key_evict=key_evict)
    if wl["model"] == "nfm":  # the dense layers as bench.py initialises them
        rng0 = np.random.default_rng(99)
        dims = [k] + list(wl["hidden"]) + [1]
        for li in range(len(dims) - 1):
            ctx.mlp_upload(li, (rng0.random((dims[li + 1], dims[li]), dtype=np.float32) - 0.5), np.zeros(dims[li + 1], np.float32))
    out = {}
    if keyed:  # rows get W = 0, V ~ N(0,1)/sqrt(k) when their key is first uploaded
        ctx.set_key_init(1234, float(1.0 / np.sqrt(k)))
        keys = [fmix64(b[1]) for b in batches]
        ctx.profile(True)
        per = {}
        for phase in ("first_sight", "all_known"):
            per[phase] = []
            for i, (rp, fid, fld, lab) in enumerate(batches):
                ctx.profile_read(reset=True)
                ctx.upload_batch_keys(i, rp, keys[i], fld if Fc else None, None, lab)
                per[phase].append(ctx.profile_read(reset=True)["keys_translate"][0])
        ctx.profile(False)
        out["translate_us_per_batch"] = {"first_sight": 1e3 * float(np.mean(per["first_sight"])),
                                         "first_batch": 1e3 * per["first_sight"][0],
                                         "all_known": 1e3 * float(np.mean(per["all_known"])), "batches": len(batches),
                                         "rows_created": int(len(ctx.download_keys()))}
        T = 16
        while T < 2 * F:
            T *= 2
        out["table_bytes"] = {"key_table": T * 12 + F * 8, "shard": ctx.device_bytes()[0]}
    else:
        ctx.fill_params(1234, float(1.0 / np.sqrt(k)))
        for i, (rp, fid, fld, lab) in enumerate(batches):
            ctx.upload_batch(i, rp, fid, fld if Fc else None, None, lab)
    stream = torch.cuda.ExternalStream(ctx.stream())
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    NB = len(batches)

    def step(i, ev=None):
        with torch.cuda.stream(stream):
            flush.zero_()
            if ev:
                ev[0].record(stream)
        ctx.train_step(i % NB, want_stats=False)
        if ev:
            with torch.cuda.stream(stream):
                ev[1].record(stream)

    for i in range(max(warmup, 3)):
        step(i)
    ctx.sync()
    evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    for i in range(steps):
        step(i, evs[i])
    ctx.sync()
    torch.cuda.synchronize()
    out["ms_per_step"] = float(np.mean([a.elapsed_time(b) for a, b in evs]))
    ctx.close()
    del flush
    torch.cuda.empty_cache()
    return out


def evict_times(wl, rounds, fractions=(0.10, 0.25, 0.50)):
    """lctr_evict_keys on a full 1M-row table with ages spread over 0..99, restored from one checkpoint before each call"""
    import ctypes as C
    from lightctr_b200 import capi
    F, k = wl["F"], wl["k"]
    ctx = capi.Context(capi.MODEL_FM, F, k, optimizer=capi.OPT_ADAGRAD, key_mode=capi.KEYS_HASHED, key_evict=True)
    ctx.set_key_init(1234, float(1.0 / np.sqrt(k)))
    keys = fmix64(np.arange(F, dtype=np.uint64) + np.uint64(1 << 40))
    ctx.upload_keyed_params(keys)  # every row, lazily initialised
    perm = np.random.default_rng(7).permutation(F)
    one = np.array([0, 1], np.int64)
    for chunk in np.array_split(perm, 100):  # one insert-upload per chunk, then that chunk is stamped with its clock
        ctx.upload_batch_keys(0, one, keys[chunk[:1]], None, None, np.array([1], np.int32))
        ctx.upload_keyed_params(keys[chunk])
    out = {"rows": F, "evict_ms": {}, "rows_moved": {}}
    kbuf, wbuf, vbuf = np.empty(F, np.uint64), np.empty(F, np.float32), np.empty(F * k, np.float32)
    n = C.c_uint64()
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "full.ckpt")
        ctx.save_checkpoint(path)
        rows0 = ctx.lookup_keys(keys)
        ctx.evict_keys(max_rows=F)  # allocates the eviction scratch; frees nothing
        for f in fractions:
            for export in (False, True):
                name = "%d%%%s" % (round(f * 100), "_export" if export else "")
                out["evict_ms"][name] = []
                for _ in range(rounds):
                    ctx.load_checkpoint(path)
                    ptrs = (kbuf.ctypes.data, wbuf.ctypes.data, vbuf.ctypes.data) if export else (None, None, None)
                    t0 = time.perf_counter()
                    rc = ctx.L.lctr_evict_keys(ctx.h, capi.NO_LIMIT, int(F * (1 - f)), *ptrs, F if export else 0, C.byref(n))
                    dt = time.perf_counter() - t0
                    if rc:
                        raise RuntimeError(capi.load_library().lctr_last_error().decode())
                    out["evict_ms"][name].append(1e3 * dt)
                rows1 = ctx.lookup_keys(keys)
                out["rows_moved"]["%d%%" % round(f * 100)] = int(np.sum((rows1 >= 0) & (rows1 != rows0)))
                out.setdefault("rows_evicted", {})["%d%%" % round(f * 100)] = int(n.value)
    ctx.close()
    return out


def main_evict(args):
    wl = dict(WORKLOADS["fm_c2"])
    batches = make_batches(wl, wl.get("nb", 8))
    line = {"workload": wl["desc"] + ", keyed capacity 1M", "keys": "key = fmix64(fid)", "gpu": gpu_info(), "steps": args.steps,
            "translate_us_per_batch": {"tracked": [], "untracked": []},
            "ms_per_step": {"dense": [], "untracked": [], "tracked": []}}
    for r in range(args.rounds):
        order = (False, True) if r % 2 == 0 else (True, False)
        for tracked in order:
            kd = run(wl, batches, True, args.steps, args.warmup, key_evict=tracked)
            name = "tracked" if tracked else "untracked"
            line["translate_us_per_batch"][name].append(kd["translate_us_per_batch"])
            line["ms_per_step"][name].append(kd["ms_per_step"])
        line["ms_per_step"]["dense"].append(run(wl, batches, False, args.steps, args.warmup)["ms_per_step"])
    line.update(evict_times(wl, max(args.rounds, 3)))
    print(json.dumps(line))
    return 0


ADMIT_LW = 22


def admit_model(key_batches, passes, min_count, lw=ADMIT_LW):
    """rows held after each pass of the stream: numpy restatement of the sketch (include/lightctr_b200.h) and the rule"""
    gold = 0x9E3779B97F4A7C15

    def cells(keys):
        return [(fmix64(keys ^ np.uint64(((i + 1) * gold) % (1 << 64))) >> np.uint64(64 - lw)).astype(np.int64) for i in range(4)]

    sk = np.zeros((4, 1 << lw), np.int64)
    present = np.zeros(0, np.uint64)
    out = []
    for _ in range(passes):
        for keys in key_batches:
            absent = keys[~np.isin(keys, present)]
            for i, c in enumerate(cells(absent)):
                sk[i] += np.bincount(c, minlength=1 << lw)
            new = np.unique(absent)
            cnt = np.min(np.stack([sk[i][c] for i, c in enumerate(cells(new))]), axis=0) if len(new) else np.zeros(0)
            present = np.union1d(present, new[cnt >= min_count])
        out.append(int(len(present)))
    return out


def admit_run(wl, batches, keys, min_count):
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_FM, wl["F"], wl["k"], optimizer=capi.OPT_ADAGRAD, max_nnz=wl["batch"] * 100,
                       key_mode=capi.KEYS_HASHED)
    ctx.set_key_init(1234, float(1.0 / np.sqrt(wl["k"])))
    ctx.set_key_admission(min_count, ADMIT_LW)
    out = {"translate_us_per_batch": {}, "upload_ms_per_batch": {}, "rows_created": [], "dropped_entries": []}
    ctx.profile(True)
    for p in ("pass1", "pass2"):
        dev, host, dropped = [], [], 0
        for i, (rp, fid, fld, lab) in enumerate(batches):
            ctx.profile_read(reset=True)
            t0 = time.perf_counter()
            rc = ctx.L.lctr_upload_batch_keys(ctx.h, i, len(rp) - 1, len(keys[i]), rp.ctypes.data, keys[i].ctypes.data, None,
                                              None, lab.ctypes.data, 1)
            host.append(1e3 * (time.perf_counter() - t0))
            if rc:
                raise RuntimeError(capi.load_library().lctr_last_error().decode())
            dev.append(1e3 * ctx.profile_read(reset=True)["keys_translate"][0])
            dropped += ctx.key_admission_stats()[0]
        out["translate_us_per_batch"][p] = float(np.mean(dev))
        out["upload_ms_per_batch"][p] = float(np.mean(host))
        out["rows_created"].append(int(len(ctx.download_keys())))
        out["dropped_entries"].append(int(dropped))
    ctx.profile(False)
    ctx.close()
    return out


def main_admit(args):
    wl = dict(WORKLOADS["fm_c2"])
    batches = make_batches(wl, wl.get("nb", 8))
    batches = [(np.ascontiguousarray(rp, np.int64), fid, fld, np.ascontiguousarray(lab, np.int32)) for rp, fid, fld, lab in batches]
    keys = [fmix64(b[1]) for b in batches]
    line = {"workload": wl["desc"] + ", keyed capacity 1M", "keys": "key = fmix64(fid)", "gpu": gpu_info(),
            "sketch": "4 x 2^%d u32" % ADMIT_LW, "batches": len(batches), "entries": int(sum(len(k) for k in keys)),
            "min_count": {}}
    names = [1, 2, 4]
    for r in range(args.rounds):
        for mc in (names if r % 2 == 0 else names[::-1]):
            o = admit_run(wl, batches, keys, mc)
            d = line["min_count"].setdefault(str(mc), {"translate_us_per_batch": {"pass1": [], "pass2": []},
                                                       "upload_ms_per_batch": {"pass1": [], "pass2": []}})
            for p in ("pass1", "pass2"):
                d["translate_us_per_batch"][p].append(o["translate_us_per_batch"][p])
                d["upload_ms_per_batch"][p].append(o["upload_ms_per_batch"][p])
            d["rows_created"], d["dropped_entries"] = o["rows_created"], o["dropped_entries"]
    for mc in names:
        line["min_count"][str(mc)]["rows_created"] = {"gpu": line["min_count"][str(mc)]["rows_created"],
                                                      "model": admit_model(keys, 2, mc)}
    print(json.dumps(line))
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="fm_c2", choices=["fm_c2", "ffm_c3", "nfm_c4"])
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2, help="dense / keyed alternations")
    ap.add_argument("--evict", action="store_true", help="row eviction (key_evict) instead: see the module docstring")
    ap.add_argument("--admit", action="store_true", help="frequency admission instead: see the module docstring")
    args = ap.parse_args()
    import torch
    from lightctr_b200 import build as lbuild
    lbuild.build()
    if not torch.cuda.is_available():
        raise SystemExit("bench_keys.py: no CUDA device (the product has no CPU path)")
    if args.evict:
        return main_evict(args)
    if args.admit:
        return main_admit(args)
    wl = dict(WORKLOADS[args.workload])
    batches = make_batches(wl, wl.get("nb", 8))
    line = {"workload": wl["desc"], "keys": "key = fmix64(fid), keyed context of capacity F", "gpu": gpu_info(),
            "steps": args.steps, "dense_ms_per_step": [], "keyed_ms_per_step": [], "translate_us_per_batch": []}
    for _ in range(args.rounds):
        d = run(wl, batches, False, args.steps, args.warmup)
        kd = run(wl, batches, True, args.steps, args.warmup)
        line["dense_ms_per_step"].append(d["ms_per_step"])
        line["keyed_ms_per_step"].append(kd["ms_per_step"])
        line["translate_us_per_batch"].append(kd["translate_us_per_batch"])
        line["table_bytes"] = kd["table_bytes"]
    print(json.dumps(line))
    return 0


if __name__ == "__main__":
    sys.exit(main())
