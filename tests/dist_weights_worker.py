"""One rank of a two-rank weighted training run (launched by tests/test_row_weights_gpu.py):

    RANK=r WORLD_SIZE=2 MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_weights_worker.py --out DIR --model M [...]

Both ranks use cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo.  The batches, W0 / V0 and the dense
layers are those of tests/multirank.py; each rank weights its own rows with weights(rank, step, rows).  Two train steps;
the losses and accuracies of the steps and the parameters after them go to rank<r>.npz / rank<r>.json."""
import argparse

import numpy as np

import multirank as mr

STEPS = 2


def weights(rank, step, rows):
    """the weights rank `rank` gives its rows at step `step`: [0, 4), every seventh row 0"""
    w = (np.random.default_rng(1000 * rank + step).random(rows) * 4).astype(np.float32)
    w[::7] = 0.0
    return w


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="fm")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--out", required=True)
    args = ap.parse_args()

    def body(rank, world):
        import torch.distributed as dist
        from lightctr_b200 import dist as ldist
        ctx = mr.make_context(args.model, args.F, args.k, rank, world, minibatch_size=world * args.rows, max_nnz=args.rows * 200)
        ctx.upload_params(*mr.make_params(args.F, args.k, args.model))
        for l, (w, b) in enumerate(mr.dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
        if args.model == "nfm":
            ldist.attach_dense_allreduce(ctx)
        ldist.connect(ctx)
        out, arrs = {"rank": rank, "loss": [], "acc": []}, {}
        for i, b in enumerate(mr.train_batches(args.F, args.rows, STEPS, rank)):
            mr.upload(ctx, args.model, 0, b)
            ctx.set_row_weights(0, weights(rank, i, len(b[3])))
            loss, acc = ctx.train_step(0)
            out["loss"].append(loss)
            out["acc"].append(acc)
        arrs["W"], arrs["V"] = ctx.download_params()
        dist.barrier()  # no peer uses this context's memory any more
        ctx.close()
        mr.save(args.out, rank, arrs, out)
        dist.barrier()
    mr.main(body, device=0)


if __name__ == "__main__":
    main()
