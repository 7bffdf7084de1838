"""One rank of a multi-process run of the collective predict (launched by tests/test_predict_dist_gpu.py):

    RANK=r WORLD_SIZE=R MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_predict_worker.py --out DIR --mode M [...]

Every rank uses cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo.  Train and test batches, W0 / V0 and the
dense layers are those of tests/multirank.py.

mode=parity     : --steps train steps on slot 0, then the rank's test batch into slot 1 and predict (--keyed: keyed FM,
                  the row -> key map saved after the predict).
mode=interleave : train, predict slot 1 twice, train, predict slots 1 and 2, train (--no-predict: the same steps without
                  the predicts); parameters after each train step and the launch count of each step.
mode=wnd        : Wide&Deep: predict, predict, train step, predict.
mode=empty      : rank 1's share is empty: predict on a test slot (not NFM: refused), then a train step from W0 / V0 (--keyed:
                  keyed FM; NFM with the dense all-reduce; Wide&Deep with per-rank dense layers).
mode=metrics    : dist.eval_global on predicted pCTR and on a crafted pCTR array, shares of --test-rows-per-rank rows, then
                  a call whose labels do not match on rank 1.
mode=refuse     : the quirk slot and NFM refused on world > 1, then a predict whose key list outgrows an inbox.
Each writes rank<r>.npz (arrays) and rank<r>.json (messages)."""
import argparse

import numpy as np

import multirank as mr


def empty_batch():
    return (np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(0, np.int32))


def context(model, F, k, rank, world, rows, **kw):
    """the context of every run here; world = 1 gives the reference context of the same configuration"""
    return mr.make_context(model, F, k, rank, world, minibatch_size=2 * rows, max_nnz=rows * 200, **kw)


def start(args, rank, world, model=None, keyed=False):
    from lightctr_b200 import dist as ldist
    model = model or args.model
    ctx = context(model, args.F, args.k, rank, world, args.rows, keyed=keyed)
    if not keyed:
        ctx.upload_params(*mr.make_params(args.F, args.k, model))
    ldist.connect(ctx)
    return ctx


def run_parity(args, rank, world, out, arrs):
    ctx = start(args, rank, world, keyed=args.keyed)
    for b in mr.train_batches(args.F, args.rows, args.steps, rank):
        mr.upload(ctx, args.model, 0, b, keyed=args.keyed)
        ctx.train_step(0)
    mr.upload(ctx, args.model, 1, mr.test_batches(args.F, args.test_rows, 1, rank)[0], keyed=args.keyed)
    arrs["pctr"] = ctx.predict(1)
    if args.keyed:  # the test upload created the rows of its unseen keys
        arrs["keys"] = ctx.download_keys()
    arrs["W"], arrs["V"] = ctx.download_params()
    return ctx


def run_interleave(args, rank, world, out, arrs):
    ctx = start(args, rank, world)
    tb = mr.train_batches(args.F, args.rows, 3, rank)
    t1, t2 = mr.test_batches(args.F, args.test_rows, 2, rank)
    launches = []

    def step(i):
        mr.upload(ctx, args.model, 0, tb[i])
        n = ctx.launch_count()
        ctx.train_step(0)
        launches.append(ctx.launch_count() - n)
        arrs["W%d" % i], arrs["V%d" % i] = ctx.download_params()

    mr.upload(ctx, args.model, 1, t1)
    mr.upload(ctx, args.model, 2, t2)
    step(0)
    if not args.no_predict:
        arrs["p1a"], arrs["p1b"] = ctx.predict(1), ctx.predict(1)
    step(1)
    if not args.no_predict:
        arrs["p2_1"], arrs["p2_2"] = ctx.predict(1), ctx.predict(2)
    step(2)
    arrs["launches"] = np.array(launches)
    return ctx


def run_wnd(args, rank, world, out, arrs):
    ctx = start(args, rank, world, model="wnd")
    for l, (w, b) in enumerate(mr.dense_layers("wnd", args.k)):
        ctx.mlp_upload(l, w, b)
    mr.upload(ctx, "wnd", 0, mr.train_batches(args.F, args.rows, 1, rank)[0])
    mr.upload(ctx, "wnd", 1, mr.test_batches(args.F, args.test_rows, 1, rank)[0])
    arrs["p1a"], arrs["p1b"] = ctx.predict(1), ctx.predict(1)
    out["loss"] = ctx.train_step(0)[0]
    arrs["p2"] = ctx.predict(1)
    return ctx


def run_empty(args, rank, world, out, arrs):
    from lightctr_b200 import dist as ldist
    ctx = start(args, rank, world, keyed=args.keyed)
    dense = args.model in ("nfm", "wnd")
    if dense:
        for l, (w, b) in enumerate(mr.dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
    if args.model == "nfm":
        ldist.attach_dense_allreduce(ctx)
    predicts = args.model != "nfm"
    share = mr.test_batches(args.F, args.test_rows, 1, rank)[0] if rank == 0 else empty_batch()
    mr.upload(ctx, args.model, 1, share, keyed=args.keyed)
    if predicts:
        arrs["pctr"] = ctx.predict(1)
    train = mr.train_batches(args.F, args.rows, 1, rank)[0] if rank == 0 else empty_batch()
    mr.upload(ctx, args.model, 0, train, keyed=args.keyed)
    loss, correct = ctx.train_step(0)
    out["stats"] = [loss, correct]
    out["reduced"] = list(ldist.reduce_stats(loss, correct))
    if predicts:
        arrs["pctr_after"] = ctx.predict(1)
    if args.keyed:
        arrs["keys"] = ctx.download_keys()
    arrs["W"], arrs["V"] = ctx.download_params()
    if dense:
        dims = mr.layer_dims(args.model, args.k)
        for l in range(len(dims) - 1):
            arrs["mlp_w%d" % l], arrs["mlp_b%d" % l] = ctx.mlp_download(l, dims[l], dims[l + 1])
    return ctx


def crafted_pctr(n, rank):
    """ties, values that share an AucEvaluator bucket (width 1 / (2^24 - 1)), and the ends of [0, 1]"""
    rng = np.random.default_rng(300 + rank)
    p = rng.random(n).astype(np.float32)
    special = np.array([0.5, 0.5, 0.25, np.nextafter(np.float32(0.25), np.float32(1)), 0.0, 1.0, 0.75, 0.75], np.float32)
    m = min(n, len(special))
    p[:m] = special[:m]
    p[m::7] = np.float32(0.125)  # many ties
    return p


def run_metrics(args, rank, world, out, arrs):
    from lightctr_b200 import dist as ldist
    ctx = start(args, rank, world)
    rows = args.test_rows_per_rank[rank]
    batch = mr.test_batches(args.F, rows, 1, rank)[0] if rows else empty_batch()
    mr.upload(ctx, args.model, 1, batch)
    arrs["pctr"] = ctx.predict(1)
    out["predicted"] = list(ldist.eval_global(ctx, 1, batch[3]))
    crafted = crafted_pctr(rows, rank)
    ctx.upload_pred(1, crafted)
    arrs["crafted"] = crafted
    out["crafted"] = list(ldist.eval_global(ctx, 1, batch[3]))
    try:  # rank 1 passes one label too few: every rank fails the call, none is left in the exchange
        ldist.eval_global(ctx, 1, batch[3][:-1] if rank == 1 else batch[3])
        out["mismatch"] = None
    except ValueError as e:
        out["mismatch"] = str(e)
    return ctx


def run_refuse(args, rank, world, out, arrs):
    import torch.distributed as dist
    from lightctr_b200 import capi, dist as ldist

    def attempt(fn):
        try:
            fn()
            return None
        except capi.LctrError as e:
            return str(e)

    ctx = start(args, rank, world)
    mr.upload(ctx, "fm", 0, mr.train_batches(args.F, args.rows, 1, rank)[0])
    mr.upload(ctx, "fm", 1, mr.test_batches(args.F, args.test_rows, 1, rank)[0])
    ctx.train_step(0)
    out["quirk"] = attempt(lambda: ctx.predict(1, quirk_sumvx_slot=0))
    arrs["after_quirk"] = ctx.predict(1)  # the refusal launched nothing: the ranks still agree on the protocol
    dist.barrier()  # no peer uses this context's memory any more
    ctx.close()
    nfm = context("nfm", args.F, args.k, rank, world, args.rows, hidden=(16,))
    ldist.connect(nfm)
    mr.upload(nfm, "nfm", 1, mr.test_batches(args.F, args.test_rows, 1, rank)[0])
    out["nfm"] = attempt(lambda: nfm.predict(1))
    dist.barrier()
    nfm.close()
    # rank 0's test batch: 20000 distinct rows all owned by rank 0, more than its inbox from rank 0 holds (3 * max_nnz /
    # (2 * world) + 4096 = 19096 records with max_nnz = 20000)
    over = context("fm", 65536, args.k, rank, world, 100)
    over.upload_params(*mr.make_params(65536, args.k, "fm"))
    ldist.connect(over)
    if rank == 0:
        fid = (2 * np.arange(20000)).astype(np.uint32)
        batch = (np.arange(0, 20001, 100).astype(np.int64), fid, None, np.zeros(200, np.int32))
    else:
        batch = mr.test_batches(65536, 100, 1, rank)[0]
    mr.upload(over, "fm", 1, batch)
    out["overflow"] = attempt(lambda: over.predict(1))
    return over


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="parity")
    ap.add_argument("--model", default="fm")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--test-rows", type=int, default=200)
    ap.add_argument("--test-rows-per-rank", type=lambda s: [int(x) for x in s.split(",")], default=[300, 170])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--no-predict", action="store_true")
    ap.add_argument("--keyed", action="store_true")
    ap.add_argument("--out", required=True)
    args = ap.parse_args()
    run = {"parity": run_parity, "interleave": run_interleave, "wnd": run_wnd, "empty": run_empty, "metrics": run_metrics,
           "refuse": run_refuse}[args.mode]

    def body(rank, world):
        import torch.distributed as dist
        out, arrs = {"rank": rank}, {}
        ctx = run(args, rank, world, out, arrs)
        dist.barrier()
        mr.save(args.out, rank, arrs, out)
        dist.barrier()
        ctx.close()
    mr.main(body, device=0)


if __name__ == "__main__":
    main()
