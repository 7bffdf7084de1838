"""One rank of a multi-process run of the keyed multi-GPU path (launched by tests/test_keyed_dist_gpu.py):

    RANK=r WORLD_SIZE=R MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_keyed_worker.py --out DIR [...]

Every rank uses cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo.  Keys are fmix64(fid) of the
CriteoSynth train batches of tests/multirank.py, rows created by lazy init or seeded with
upload_keyed_params (--seeded: the same arrays on every rank).

mode=train : --steps collective uploads + steps; writes rank<r>.npz with the rank's row -> key map, its download_params
             arrays, the global rows lookup_keys gives for them and the reduced per-step (loss, correct).
mode=edge  : FM on a tiny capacity: a batch overflowing one owner's shard, refused uploads (insert = 0, and on one rank
             only), recovery after each, and key_evict or a missing max_nnz refused with world > 1; writes rank<r>.json with what happened."""
import argparse

import numpy as np

import multirank as mr


def run_train(args, rank, world):
    import torch.distributed as dist
    from lightctr_b200 import dist as ldist
    ctx = mr.make_context(args.model, args.F, args.k, rank, world, minibatch_size=world * args.rows,
                          max_nnz=args.rows * 200, keyed=True)
    ldist.connect(ctx)
    if args.seeded:
        ctx.upload_keyed_params(ldist.fmix64(np.arange(args.F)), *mr.make_params(args.F, args.k, args.model))
    if args.model == "nfm":
        for l, (w, b) in enumerate(mr.dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
        ldist.attach_dense_allreduce(ctx)
    stats = []
    for b in mr.train_batches(args.F, args.rows, args.steps, rank):
        mr.upload(ctx, args.model, 0, b, keyed=True)
        l, c = ctx.train_step(0)
        stats.append(ldist.reduce_stats(l, c))
    dist.barrier()
    keys = ctx.download_keys()
    W, V = ctx.download_params()
    mr.save(args.out, rank, dict(keys=keys, W=W, V=V, rows=ctx.lookup_keys(keys), stats=np.array(stats),
                                 launches=ctx.launch_count()))
    dist.barrier()
    ctx.close()


def _csr(rows_of_keys, seed):
    rp = np.concatenate([[0], np.cumsum([len(r) for r in rows_of_keys])]).astype(np.int64)
    keys = np.concatenate(rows_of_keys).astype(np.uint64)
    lab = (np.random.default_rng(seed).random(len(rows_of_keys)) < 0.3).astype(np.int32)
    return rp, keys, lab


def run_edge(args, rank, world):
    import torch.distributed as dist
    from lightctr_b200 import capi, dist as ldist
    k, rows, cap = 8, 16, 64  # each rank's shard holds 32 rows
    out = {"rank": rank}
    try:
        capi.Context(capi.MODEL_FM, cap, k, device=0, rank=rank, world=world, minibatch_size=world * rows,
                     max_nnz=rows * 200, key_mode=capi.KEYS_HASHED, key_evict=True)
        out["evict_create"] = None
    except capi.LctrError as e:
        out["evict_create"] = str(e)
    try:
        capi.Context(capi.MODEL_FM, cap, k, device=0, rank=rank, world=world, minibatch_size=world * rows,
                     key_mode=capi.KEYS_HASHED)
        out["no_max_nnz_create"] = None
    except capi.LctrError as e:
        out["no_max_nnz_create"] = str(e)
    ctx = mr.make_context("fm", 0, k, rank, world, minibatch_size=world * rows, max_nnz=rows * 200, keyed=True, cap=cap)
    ldist.connect(ctx)
    pool = ldist.fmix64(np.arange(1, 20000))
    own = [pool[ldist.owner_of_key(pool, world) == o] for o in range(world)]
    # batch A: 10 keys of each owner, every row 5 keys
    a_keys = np.concatenate([own[0][:10], own[1][:10]])
    rng = np.random.default_rng(rank)
    batch_a = _csr([rng.choice(a_keys, 5, replace=False) for _ in range(rows)], 10 + rank)

    def upload(b, insert=True):
        try:
            ctx.upload_batch_keys(0, b[0], b[1], None, None, b[2], insert=insert)
            return None
        except capi.LctrError as e:
            return str(e)

    def step():
        try:
            return ctx.train_step(0)[0]
        except capi.LctrError as e:
            return str(e)

    out["a_upload"] = upload(batch_a)
    out["a_loss"] = step()
    known = ctx.lookup_keys(a_keys)
    out["rows_after_a"] = int(len(ctx.download_keys()))
    # batch B: rank 0 brings 30 new keys of owner 1 (its shard has 32 rows, batch A took up to 10), rank 1 only known keys
    # of owner 0
    if rank == 0:
        batch_b = _csr([own[1][10 + 5 * i:15 + 5 * i] for i in range(6)], 20)
    else:
        batch_b = _csr([own[0][:5] for _ in range(10)], 21)
    out["b_upload"] = upload(batch_b)
    out["b_step"] = step()
    out["kept_rows"] = bool(np.array_equal(ctx.lookup_keys(a_keys), known))
    out["rows_after_b"] = int(len(ctx.download_keys()))
    out["c_upload"] = upload(batch_a)
    out["c_loss"] = step()
    # refusals: insert = 0 on every rank, then on rank 0 only; the upload after them still works
    out["lookup_upload"] = upload(batch_a, insert=False)
    out["mixed_upload"] = upload(batch_a, insert=(rank != 0))
    out["d_upload"] = upload(batch_a)
    out["d_loss"] = step()
    dist.barrier()
    mr.save(args.out, rank, messages=out)
    dist.barrier()
    ctx.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="train")
    ap.add_argument("--model", default="fm")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--seeded", action="store_true")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    run = run_train if args.mode == "train" else run_edge
    mr.main(lambda rank, world: run(args, rank, world), device=0)


if __name__ == "__main__":
    main()
