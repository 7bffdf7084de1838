"""One rank of a multi-process run of the collective score (launched by tests/test_score_dist_gpu.py):

    RANK=r WORLD_SIZE=R MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_score_worker.py --out DIR --model M [...]

Every rank uses cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo.  Train and test batches, W0 / V0 and the
dense layers are those of tests/multirank.py (--bf16: NFM on the tensor cores with hidden layers 128, 64).

Three train steps on slot 0, each scored before it runs (s<i>) and its pred read back after it (p<i>).  After step 1 the
rank's test batch (slot 1; --empty: rank 1's share is empty) is scored and evaluated with dist.eval_global, and the
parameters and dense layers are saved.  Then the same steps run again on a fresh context without any score: losses and
parameters of both runs are saved.  Each writes rank<r>.npz (arrays) and rank<r>.json (numbers)."""
import argparse

import numpy as np

import multirank as mr

BF16_HIDDEN = (128, 64)


def empty_batch():
    return (np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(0, np.int32))


def context(args, rank, world):
    """the context of every run here; world = 1 gives the reference context of the same configuration"""
    from lightctr_b200 import capi
    kw = dict(hidden=BF16_HIDDEN, mlp_precision=capi.MLP_BF16) if args.bf16 else {}
    return mr.make_context(args.model, args.F, args.k, rank, world, minibatch_size=2 * args.rows, max_nnz=args.rows * 200,
                           keyed=args.keyed, **kw)


def dense_layers(args):
    if not args.bf16:
        return mr.dense_layers(args.model, args.k)
    rng = np.random.default_rng(78)
    dims = [args.k] + list(BF16_HIDDEN) + [1]
    return [((rng.random((dims[i + 1], dims[i]), dtype=np.float32) - 0.5) / np.float32(np.sqrt(dims[i] / 12.0)),
             np.zeros(dims[i + 1], np.float32)) for i in range(len(dims) - 1)]


def layer_dims(args):
    return [args.k] + list(BF16_HIDDEN) + [1] if args.bf16 else mr.layer_dims(args.model, args.k)


def run(args, rank, world, out, arrs, score):
    from lightctr_b200 import dist as ldist
    ctx = context(args, rank, world)
    if not args.keyed:
        ctx.upload_params(*mr.make_params(args.F, args.k, args.model))
    for l, (w, b) in enumerate(dense_layers(args) if args.model in ("nfm", "wnd") else []):
        ctx.mlp_upload(l, w.astype(np.float32), b)
    if args.model == "nfm":
        ldist.attach_dense_allreduce(ctx)
    ldist.connect(ctx)
    test = mr.test_batches(args.F, args.test_rows, 1, rank)[0] if not (args.empty and rank == 1) else empty_batch()
    mr.upload(ctx, args.model, 1, test, keyed=args.keyed)
    tag = "" if score else "n_"
    losses = []
    for i, b in enumerate(mr.train_batches(args.F, args.rows, 3, rank)):
        mr.upload(ctx, args.model, 0, b, keyed=args.keyed)
        if score:
            arrs["s%d" % i] = ctx.score(0)
        losses.append(ctx.train_step(0)[0])
        if score:
            arrs["p%d" % i] = ctx.download_pred(0)
        if score and i == 1:
            arrs["test"] = ctx.score(1)
            arrs["test_label"] = test[3]
            out["eval"] = list(ldist.eval_global(ctx, 1, test[3]))
            arrs["W"], arrs["V"] = ctx.download_params()
            dims = layer_dims(args)
            for l in range(len(dims) - 1):
                arrs["mlp_w%d" % l], arrs["mlp_b%d" % l] = ctx.mlp_download(l, dims[l], dims[l + 1])
    out[tag + "loss"] = losses
    if not args.keyed:
        arrs[tag + "W_end"], arrs[tag + "V_end"] = ctx.download_params()
    return ctx


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default="fm")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--test-rows", type=int, default=200)
    ap.add_argument("--bf16", action="store_true")
    ap.add_argument("--keyed", action="store_true")
    ap.add_argument("--empty", action="store_true")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()

    def body(rank, world):
        import torch.distributed as dist
        out, arrs = {"rank": rank}, {}
        for score in (True, False):
            ctx = run(args, rank, world, out, arrs, score)
            dist.barrier()  # no peer uses this context's memory any more
            ctx.close()
        mr.save(args.out, rank, arrs, out)
        dist.barrier()
    mr.main(body, device=0)


if __name__ == "__main__":
    main()
