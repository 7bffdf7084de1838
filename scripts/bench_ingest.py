#!/usr/bin/env python
"""scripts/bench_ingest.py -- libffm text into a batch slot on the device (lctr_upload_libffm) against the host loader.

    python scripts/bench_ingest.py [--batches 8] [--reps 5]

The text is C2's synthetic batches (bench.py fm_c2: 4096 rows of ~77 entries, about 1 KB of text per row) written in the
reference's libffm format, one 4096-row chunk per batch.  In one process, one JSON line:
  host_*    lctr_load_libffm on the whole text (a temporary file): MB/s and rows/s;
  upload_*  lctr_upload_libffm per 4096-row chunk from pinned memory, host clock around the call (which ends in a stream
            synchronise): ms per chunk (median), rows/s and MB/s;
  parse_*   the parse kernels alone (the library's per-launch events, a run of its own): ms per chunk and text GB/s;
  h2d_*     a host-to-device copy of one chunk from pinned memory (CUDA events): ms and GB/s;
  train_*   text -> slot -> lctr_train_step per chunk, FM k = 16 on 1M features: samples/s;
and the card's name, power limit and max SM clock, read in the same run.
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

import numpy as np  # noqa: E402

from bench import WORKLOADS, make_batches  # noqa: E402


def chunk_text(rp, fid, fld, lab):
    rows = []
    for r in range(len(rp) - 1):
        b, e = rp[r], rp[r + 1]
        rows.append("%d\t%s\n" % (lab[r], " ".join("%d:%d:1" % (fld[i], fid[i]) for i in range(b, e))))
    return "".join(rows).encode()


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, power, clock = (s.strip() for s in q.stdout.strip().split(","))
    return dict(gpu=name, power_limit=power, max_sm_clock=clock)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=8)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    from lightctr_b200 import build as lbuild
    from lightctr_b200 import capi
    if not torch.cuda.is_available():
        raise SystemExit("bench_ingest: no CUDA device")
    lbuild.build()
    wl = WORKLOADS["fm_c2"]
    chunks = [chunk_text(rp, fid, fld, lab) for rp, fid, fld, lab in make_batches(wl, args.batches)]
    rows_per = [c.count(b"\n") for c in chunks]
    total = sum(len(c) for c in chunks)
    out = dict(workload="fm_c2 batches as libffm text", chunks=len(chunks), rows_per_chunk=rows_per[0],
               bytes_per_row=round(total / sum(rows_per), 1), **card())

    # host loader
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "c2.txt")
        with open(path, "wb") as f:
            for c in chunks:
                f.write(c)
        capi.load_libffm(path)  # warm the page cache
        t0 = time.perf_counter()
        ds = capi.load_libffm(path)
        secs = time.perf_counter() - t0
    out.update(host_MBps=round(total / secs / 1e6, 1), host_rows_per_s=round(ds.rows / secs))

    # pinned chunks
    pinned = torch.empty(total, dtype=torch.uint8).pin_memory()
    host = pinned.numpy()
    offs = np.cumsum([0] + [len(c) for c in chunks])
    for c, o in zip(chunks, offs):
        host[o:o + len(c)] = np.frombuffer(c, np.uint8)
    views = [host[o:o + len(c)] for c, o in zip(chunks, offs)]

    ctx = capi.Context(capi.MODEL_FM, wl["F"], wl["k"], minibatch_size=wl["batch"])
    ctx.fill_params(1, 0.01)
    for v in views:  # warm-up: staging buffers, slot capacity, module load
        info = ctx.upload_libffm(0, v)
        assert info.host_lines == 0 and info.rows == wl["batch"]
    ms = []
    for _ in range(args.reps):
        for v in views:
            t0 = time.perf_counter()
            ctx.upload_libffm(0, v)
            ms.append(1e3 * (time.perf_counter() - t0))
    up = float(np.median(ms))
    per_chunk_bytes = total / len(chunks)
    out.update(upload_ms_per_chunk=round(up, 3), upload_rows_per_s=round(rows_per[0] / up * 1e3),
               upload_MBps=round(per_chunk_bytes / up / 1e3, 1))
    out["speedup_rows_per_s"] = round(out["upload_rows_per_s"] / out["host_rows_per_s"], 1)

    # parse kernels alone (events around the parse launches; a run of its own)
    ctx.profile(True)
    ctx.profile_read(reset=True)
    for _ in range(args.reps):
        for v in views:
            ctx.upload_libffm(0, v)
    prof = ctx.profile_read(reset=True)
    ctx.profile(False)
    parse_ms = prof["text_parse"][0] / (args.reps * len(views))
    out.update(parse_ms_per_chunk=round(parse_ms, 4), parse_GBps=round(per_chunk_bytes / parse_ms / 1e6, 1))

    # host -> device copy of one chunk
    dst = torch.empty(len(chunks[0]), dtype=torch.uint8, device="cuda")
    src = pinned[:len(chunks[0])]
    for _ in range(3):
        dst.copy_(src, non_blocking=True)
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 50
    a.record()
    for _ in range(n):
        dst.copy_(src, non_blocking=True)
    b.record()
    torch.cuda.synchronize()
    h2d = a.elapsed_time(b) / n
    out.update(h2d_ms_per_chunk=round(h2d, 4), h2d_GBps=round(len(chunks[0]) / h2d / 1e6, 1))

    # text -> train
    for v in views:
        ctx.upload_libffm(0, v)
        ctx.train_step(0, want_stats=False)
    ctx.sync()
    t0 = time.perf_counter()
    for _ in range(args.reps):
        for v in views:
            ctx.upload_libffm(0, v)
            ctx.train_step(0, want_stats=False)
    ctx.sync()
    secs = time.perf_counter() - t0
    out.update(train_samples_per_s=round(args.reps * sum(rows_per) / secs))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
