#!/usr/bin/env python
"""Keyed against dense mode on several GPUs (csrc/dist.cu): the same CriteoSynth batches, fed to a sharded keyed context as
keys fmix64(fid) and to a sharded dense context as fids, alternated round by round in every rank.

    python -m torch.distributed.run --nproc-per-node R --master-addr 127.0.0.1 scripts/bench_keys_dist.py \\
        [--F N] [--k K] [--rows B] [--steps S] [--rounds N] [--same-device]

Rank 0 prints ONE JSON line with, per rank and per round:
  keyed_ms_per_step / dense_ms_per_step   device time of a step (a CUDA-event pair on the context's stream around each
                                          train_step, averaged over --steps steps; the steps of the ranks are collective);
  keyed_upload_ms                         host clock around the collective keyed upload of one batch (dedupe, slot map,
                                          keyed send, owner translation and the status round trip; it ends in a stream
                                          synchronise), averaged over the batches of the round;
  gpu                                     card name and power limit of each rank, read in the same run.
--same-device puts every rank on cuda:0 (CUDA IPC between processes on one GPU): the ranks then time-slice one device,
so the run checks the path end to end and its numbers are not a multi-GPU measurement.  Writes nothing to the tree.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.dont_write_bytecode = True  # the tree may be read-only

import numpy as np  # noqa: E402


def gpu_info(dev):
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(dev), "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--F", type=int, default=1 << 20)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=4096, help="rows per rank and step")
    ap.add_argument("--batches", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--same-device", action="store_true")
    args = ap.parse_args()
    import torch
    import torch.distributed as dist
    from lightctr_b200 import capi, dist as ldist
    from lightctr_b200.data import CriteoSynth
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = 0 if args.same_device else int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    gen = CriteoSynth(args.F, seed=100 + rank)
    batches = [gen.batch(args.rows) for _ in range(args.batches)]
    keys = [ldist.fmix64(b[1]) for b in batches]
    common = dict(device=dev, rank=rank, world=world, minibatch_size=world * args.rows, max_nnz=args.rows * 100)
    ctxs = {"dense": capi.Context(capi.MODEL_FM, args.F, args.k, **common),
            "keyed": capi.Context(capi.MODEL_FM, args.F, args.k, key_mode=capi.KEYS_HASHED, **common)}
    ctxs["dense"].fill_params(1234, float(1.0 / np.sqrt(args.k)))
    ctxs["keyed"].set_key_init(1234, float(1.0 / np.sqrt(args.k)))
    for c in ctxs.values():
        ldist.connect(c)

    def upload(name, i):
        c = ctxs[name]
        rp, fid, _fld, lab = batches[i]
        if name == "keyed":
            c.upload_batch_keys(i, rp, keys[i], None, None, lab)
        else:
            c.upload_batch(i, rp, fid, None, None, lab)

    for name in ctxs:  # first sight of every key: rows are created here, outside the timed rounds
        for i in range(len(batches)):
            upload(name, i)

    def steps(name):
        c = ctxs[name]
        stream = torch.cuda.ExternalStream(c.stream())
        evs = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(args.steps)]
        for i in range(args.steps):
            with torch.cuda.stream(stream):
                evs[i][0].record(stream)
            c.train_step(i % len(batches), want_stats=False)
            with torch.cuda.stream(stream):
                evs[i][1].record(stream)
        c.sync()
        return float(np.mean([a.elapsed_time(b) for a, b in evs]))

    res = {"keyed_ms_per_step": [], "dense_ms_per_step": [], "keyed_upload_ms": []}
    for _ in range(args.rounds):
        dist.barrier()
        t0 = time.perf_counter()
        for i in range(len(batches)):
            upload("keyed", i)
        res["keyed_upload_ms"].append(1e3 * (time.perf_counter() - t0) / len(batches))
        for i in range(len(batches)):  # so that both contexts' first steps rebuild the owner-side union of each slot
            upload("dense", i)
        for name in ("keyed", "dense"):
            dist.barrier()
            res[name + "_ms_per_step"].append(steps(name))
    res["gpu"] = gpu_info(dev)
    res["rows_per_rank"] = args.rows
    res["shard_rows"] = int(len(ctxs["keyed"].download_keys()))
    allres = [None] * world
    dist.all_gather_object(allres, res)
    dist.barrier()
    for c in ctxs.values():
        c.close()
    if rank == 0:
        print(json.dumps({"world": world, "same_device": args.same_device, "F": args.F, "k": args.k, "per_rank": allres}))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
