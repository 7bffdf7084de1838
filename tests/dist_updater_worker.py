"""One rank of the two-rank updater check of tests/test_updaters_gpu.py: every rule on the owner-side appliers of the
multi-GPU exchange, on the exact batches of tests/exact_batch.py.

    RANK=r WORLD_SIZE=2 MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_updater_worker.py --out DIR --k K

Both ranks share cuda:0 (IPC between processes).  k in {4, 8, 16, 32} takes the order-free path (push, then
merge_apply_kernel); any other k the dense one (push, merge_kernel, then the sparse apply_kernel).  For each rule: a
context, then three steps, each from freshly uploaded dyadic parameters with the updater state left on the device; after
each step the rank saves its shard of W, V, s1 and s2 (rank<r>.npz: <rule>_<what><step>)."""
import argparse

import numpy as np

import exact_batch as eb
import multirank as mr

F = 3000
STEPS = 3


def rank_batch(k, rows, rule, rank):
    """rank's part of the batch: the same hot and single-entry-only ids on both ranks, its own rows"""
    return eb.make_batch(500 + 10 * k + rank, F, k, rows=rows, scale=eb.SCALE[rule])


def step_params(b0, step):
    return eb.make_params(b0, 900 + 100 * step)


def union(parts):
    """the ranks' batches joined in rank order: the batch a one-GPU step would train on"""
    rp, fid, fld, lab = mr.global_batch([(b.rp, b.fid, b.fld, b.lab) for b in parts])
    u = eb.Batch(**{n: getattr(parts[0], n) for n in ("F", "k", "Fc", "scale", "l2", "single_only", "hot")})
    u.rp, u.fid, u.fld, u.lab = rp, fid, fld, lab
    u.val = np.concatenate([b.val for b in parts])
    return u


def run(args, rank, world):
    import torch
    import torch.distributed as dist
    from lightctr_b200 import dist as ldist
    torch.cuda.set_device(0)
    out = {}
    for rule in eb.RULES:
        b = rank_batch(args.k, args.rows, rule, rank)
        h = eb.HYPER
        ctx = mr.make_context("fm", F, args.k, rank, world, minibatch_size=world * args.rows, max_nnz=4 * len(b.fid),
                              device=0, optimizer=eb.capi_opt(rule), lr=h["lr"], l2=b.l2, momentum=h["beta1"],
                              momentum_adam2=h["beta2"], ema_rate=h["ema"])
        ldist.connect(ctx)
        s1, s2 = eb.make_state(rank_batch(args.k, args.rows, rule, 0), rule, 7)
        ctx.upload_opt_state(s1, s2)
        ctx.upload_batch(0, b.rp, b.fid, None, b.val, b.lab)
        for step in range(STEPS):
            W, V = step_params(rank_batch(args.k, args.rows, rule, 0), step)
            dist.barrier()  # the peer's previous step has stopped reading my shard
            ctx.upload_params(W, V)
            ctx.sync()
            dist.barrier()  # every shard holds this step's parameters
            ctx.train_step(0)
            Wg, Vg = ctx.download_params()
            a, c = ctx.download_opt_state()
            out.update({"%s_W%d" % (rule, step): Wg, "%s_V%d" % (rule, step): Vg, "%s_s1%d" % (rule, step): a,
                        "%s_s2%d" % (rule, step): c})
        dist.barrier()
        ctx.close()
        dist.barrier()
    mr.save(args.out, rank, out)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--k", type=int, default=8)
    ap.add_argument("--rows", type=int, default=150)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    mr.main(lambda rank, world: run(args, rank, world))


if __name__ == "__main__":
    main()
