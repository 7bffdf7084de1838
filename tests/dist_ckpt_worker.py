"""One rank of a multi-process run of the checkpoints of sharded trainers (launched by tests/test_ckpt_dist_gpu.py):

    RANK=r WORLD_SIZE=R MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_ckpt_worker.py --out DIR --mode M [...]

Every rank uses cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo; batches are the CriteoSynth train
batches of tests/multirank.py, keyed runs use key = fmix64(fid).

mode=resume : 6 uninterrupted steps, then 3 steps + save_sharded + fresh contexts (create, connect, load_sharded, upload
              again) + 3 steps; writes rank<r>.npz with both runs' per-step stats and final global downloads (params, optimizer
              state, keys, dense layers), and saves the final state as the set DIR/final.
mode=from1  : load_checkpoint_shards([--single]) of a single-GPU file; writes the global downloads, keys and the rows
              lookup_keys gives for --single's keys, then checks that a resident keyed slot is stale until uploaded again and
              that a collective upload + step runs on the loaded state.
mode=refuse : the refused loads, each followed by downloads equal to the ones before it; writes rank<r>.json."""
import argparse
import os

import numpy as np

import multirank as mr

HALF = 3  # resume: steps before the save


def context(args, rank, world, **kw):
    """the context of every run here; world = 1 gives its single-GPU twin"""
    return mr.make_context(args.model, args.F, args.k, rank, world, minibatch_size=2 * args.rows,
                           max_nnz=args.rows * 200, optimizer=args.opt, keyed=args.keyed, **kw)


def train(ctx, args, batches):
    from lightctr_b200 import dist as ldist
    stats = []
    for b in batches:
        mr.upload(ctx, args.model, 0, b, args.keyed)
        stats.append(ldist.reduce_stats(*ctx.train_step(0)))
    return stats


def snapshot(ctx, args):
    """global downloads of the context; with world > 1 only the rows the rank owns are filled in, the others read 0"""
    W, V = ctx.download_params()
    s1, s2 = ctx.download_opt_state()
    R, F = ctx.cfg.world, len(W)
    if R > 1:
        other = np.arange(F) % R != ctx.cfg.rank
        W[other] = 0
        V.reshape(F, -1)[other] = 0
        for s in (s1, s2):
            s[:F][other] = 0
            s[F:].reshape(F, -1)[other] = 0
    out = {"W": W, "V": V, "s1": s1, "s2": s2}
    if args.keyed:
        out["keys"] = ctx.download_keys()
    dims = mr.layer_dims(args.model, args.k)
    for l in range(len(dims) - 1):
        out["mlp_w%d" % l], out["mlp_b%d" % l] = ctx.mlp_download(l, dims[l], dims[l + 1])
    return out


def same(a, b):
    return set(a) == set(b) and all(np.array_equal(a[x], b[x]) for x in a)


def fresh(args, rank, world, W0=None, V0=None):
    from lightctr_b200 import dist as ldist
    ctx = context(args, rank, world)
    ldist.connect(ctx)
    if args.model == "nfm":
        ldist.attach_dense_allreduce(ctx)
    if W0 is not None and not args.keyed:
        ctx.upload_params(W0, V0)
    if W0 is not None:
        for l, (w, b) in enumerate(mr.dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
    return ctx


def run_resume(args, rank, world):
    import torch.distributed as dist
    from lightctr_b200 import dist as ldist
    batches, (W0, V0) = mr.train_batches(args.F, args.rows, 2 * HALF, rank), mr.make_params(args.F, args.k, args.model)
    ctx = fresh(args, rank, world, W0, V0)
    stats_a = train(ctx, args, batches)
    snap_a = snapshot(ctx, args)
    dist.barrier()
    ctx.close()
    ctx = fresh(args, rank, world, W0, V0)
    stats_b = train(ctx, args, batches[:HALF])
    prefix = os.path.join(args.out, "half")
    ldist.save_sharded(ctx, prefix)
    snap_saved = snapshot(ctx, args)
    ctx.close()
    ctx = fresh(args, rank, world)
    assert ldist.load_sharded(ctx, prefix) == world
    round_trip = same(snap_saved, snapshot(ctx, args))
    stats_b += train(ctx, args, batches[HALF:])
    snap_b = snapshot(ctx, args)
    ldist.save_sharded(ctx, os.path.join(args.out, "final"))
    mr.save(args.out, rank, dict(stats_a=np.array(stats_a), stats_b=np.array(stats_b), round_trip=round_trip,
                                 **{"a_" + x: v for x, v in snap_a.items()}, **{"b_" + x: v for x, v in snap_b.items()}))
    dist.barrier()
    ctx.close()


def run_from1(args, rank, world):
    import torch.distributed as dist
    from lightctr_b200 import capi, dist as ldist
    batches = mr.train_batches(args.F, args.rows, 2, rank)
    ctx = fresh(args, rank, world)
    out = {}
    if args.keyed:  # slot 1 holds a translated batch before the load
        mr.upload(ctx, args.model, 1, batches[0], args.keyed)
    ctx.load_checkpoint_shards([args.single])
    snap = snapshot(ctx, args)
    if args.keyed:
        snap["rows"] = ctx.lookup_keys(np.load(args.single + ".keys.npy"))
        try:
            ctx.train_step(1)
            out["stale"] = None
        except capi.LctrError as e:
            out["stale"] = str(e)
        mr.upload(ctx, args.model, 1, batches[1], args.keyed)
        out["after_upload"] = ldist.reduce_stats(*ctx.train_step(1))[0]
    else:
        out["after_upload"] = train(ctx, args, batches[:1])[0][0]
    mr.save(args.out, rank, snap, out)
    dist.barrier()
    ctx.close()


def refused(ctx, args, call):
    """call() must fail and leave the context's downloads as they were: the message, or a note of what went wrong"""
    from lightctr_b200 import capi
    before = snapshot(ctx, args)
    try:
        call()
        return "NOT REFUSED"
    except capi.LctrError as e:
        msg = str(e)
    return msg if same(before, snapshot(ctx, args)) else "CHANGED: " + msg


def run_refuse(args, rank, world):
    import torch.distributed as dist
    from lightctr_b200 import dist as ldist
    out = {"rank": rank}
    other = 1 - rank
    # dense FM: sets A (1 step) and B (2 steps)
    batches, (W0, V0) = mr.train_batches(args.F, args.rows, 2 * HALF, rank), mr.make_params(args.F, args.k, args.model)
    ctx = fresh(args, rank, world, W0, V0)
    train(ctx, args, batches[:1])
    a = os.path.join(args.out, "A")
    ldist.save_sharded(ctx, a)
    train(ctx, args, batches[1:2])
    b = os.path.join(args.out, "B")
    ldist.save_sharded(ctx, b)
    sp = ldist.shard_path
    out["other_rank"] = refused(ctx, args, lambda: ctx.load_checkpoint(sp(a, other, 2)))
    out["single_file"] = refused(ctx, args, lambda: ctx.load_checkpoint(args.single))
    out["incomplete"] = refused(ctx, args, lambda: ctx.load_checkpoint_shards([sp(a, rank, 2)]))
    out["duplicate"] = refused(ctx, args, lambda: ctx.load_checkpoint_shards([sp(a, 0, 2), sp(a, 0, 2)]))
    out["steps"] = refused(ctx, args, lambda: ctx.load_checkpoint_shards([sp(a, 0, 2), sp(b, 1, 2)]))
    out["cfg"] = refused(ctx, args, lambda: ctx.load_checkpoint_shards([args.other_cfg]))
    ctx.load_checkpoint(sp(a, rank, 2))  # the own file loads, and training goes on from it
    out["after_load"] = train(ctx, args, batches[1:2])[0][0]
    dist.barrier()
    ctx.close()
    # Wide&Deep without a dense all-reduce: per-rank layers, which a world-1 context refuses
    wargs = argparse.Namespace(**dict(vars(args), model="wnd", k=4, keyed=False))
    wb = mr.train_batches(args.F, args.rows, 1, rank)
    ctx = context(wargs, rank, world)
    ldist.connect(ctx)
    for l, (w, bb) in enumerate(mr.dense_layers("wnd", wargs.k)):
        ctx.mlp_upload(l, w, bb)
    train(ctx, wargs, wb[:1])
    wp = os.path.join(args.out, "W")
    ldist.save_sharded(ctx, wp)
    ctx1 = context(wargs, 0, 1)
    out["wnd_layers"] = refused(ctx1, wargs, lambda: ctx1.load_checkpoint_shards([sp(wp, 0, 2), sp(wp, 1, 2)]))
    ctx1.close()
    dist.barrier()
    ctx.close()
    # keyed: a single-GPU file whose keys all belong to rank 1 under world 2 overflows rank 1's shard
    kargs = argparse.Namespace(**dict(vars(args), keyed=True, k=8))
    ctx = context(kargs, rank, world, cap=64)
    ldist.connect(ctx)
    pool = ldist.fmix64(np.arange(1, 2000))
    ctx.upload_keyed_params(pool[:6], np.ones(6, np.float32), None)  # each rank seeds the keys of the 6 it owns
    out["keyed_overflow"] = refused(ctx, kargs, lambda: ctx.load_checkpoint_shards([args.skewed]))
    dist.barrier()
    ctx.close()
    mr.save(args.out, rank, messages=out)
    dist.barrier()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="resume")
    ap.add_argument("--model", default="fm")
    ap.add_argument("--opt", type=int, default=0)
    ap.add_argument("--keyed", action="store_true")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--single", default="")
    ap.add_argument("--other-cfg", default="")
    ap.add_argument("--skewed", default="")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    run = {"resume": run_resume, "from1": run_from1, "refuse": run_refuse}[args.mode]
    mr.main(lambda rank, world: run(args, rank, world), device=0)


if __name__ == "__main__":
    main()
