"""One rank of the two-rank weighted pipeline runs (launched by tests/test_weighted_stream_gpu.py):

    RANK=r WORLD_SIZE=2 MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_weighted_stream_worker.py --out DIR --mode M [...]

Both ranks use cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo; batches, W0 / V0 and the dense layers
are those of tests/multirank.py.
mode=stream  : STEPS weighted batches through lctr_train_batch_weighted_async, each rank weighting its own rows with
               weights(rank, step, rows); the lctr_wait statistics and the parameters after them.
mode=metrics : a test batch of --test-rows-per-rank rows predicted, then dist.eval_global with weights(rank, 9, rows), and a
               call with one weight too many on rank 1.
Each writes rank<r>.npz (arrays) and rank<r>.json (messages)."""
import argparse

import numpy as np

import multirank as mr

STEPS = 4


def weights(rank, step, rows):
    """the weights rank `rank` gives its rows at step `step`: [0, 4), every seventh row 0"""
    w = (np.random.default_rng(5000 + 1000 * rank + step).random(rows) * 4).astype(np.float32)
    w[::7] = 0.0
    return w


def empty_batch():
    return (np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(0, np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="stream")
    ap.add_argument("--model", default="fm")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--test-rows-per-rank", default="300,0")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()

    def body(rank, world):
        import torch.distributed as dist
        from lightctr_b200 import dist as ldist
        ctx = mr.make_context(args.model, args.F, args.k, rank, world, minibatch_size=world * args.rows,
                              max_nnz=args.rows * 200)
        ctx.upload_params(*mr.make_params(args.F, args.k, args.model))
        for l, (w, b) in enumerate(mr.dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
        if args.model == "nfm":
            ldist.attach_dense_allreduce(ctx)
        ldist.connect(ctx)
        out, arrs = {"rank": rank}, {}
        if args.mode == "stream":
            batches = mr.train_batches(args.F, args.rows, STEPS, rank)
            ws = [weights(rank, i, len(b[3])) for i, b in enumerate(batches)]  # alive until waited for
            fc = mr.field_cnt(args.model)
            tickets = [ctx.train_batch_async(b[0], b[1], b[2] if fc else None, None, b[3], weight=w)
                       for b, w in zip(batches[:2], ws[:2])]
            stats = [ctx.wait(tickets[0])]
            for b, w in zip(batches[2:], ws[2:]):
                tickets.append(ctx.train_batch_async(b[0], b[1], b[2] if fc else None, None, b[3], weight=w))
            stats += [ctx.wait(t) for t in tickets[1:]]
            out["loss"], out["acc"] = [s[0] for s in stats], [s[1] for s in stats]
            arrs["W"], arrs["V"] = ctx.download_params()
            for l, _ in enumerate(mr.dense_layers(args.model, args.k)):
                dims = mr.layer_dims(args.model, args.k)
                arrs["mlp_w%d" % l], arrs["mlp_b%d" % l] = ctx.mlp_download(l, dims[l], dims[l + 1])
        else:
            rows = [int(x) for x in args.test_rows_per_rank.split(",")][rank]
            batch = mr.test_batches(args.F, rows, 1, rank)[0] if rows else empty_batch()
            mr.upload(ctx, args.model, 1, batch)
            arrs["pctr"] = ctx.predict(1)
            arrs["label"] = batch[3]
            arrs["weight"] = weights(rank, 9, rows)
            out["metrics"] = list(ldist.eval_global(ctx, 1, batch[3], weights=arrs["weight"]))
            try:  # rank 1 passes one weight too many: every rank fails the call, none is left in the exchange
                extra = np.concatenate([arrs["weight"], np.ones(1, np.float32)])
                ldist.eval_global(ctx, 1, batch[3], weights=extra if rank == 1 else arrs["weight"])
                out["mismatch"] = None
            except ValueError as e:
                out["mismatch"] = str(e)
        dist.barrier()  # no peer uses this context's memory any more
        ctx.close()
        mr.save(args.out, rank, arrs, out)
        dist.barrier()
    mr.main(body, device=0)


if __name__ == "__main__":
    main()
