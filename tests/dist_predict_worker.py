"""One rank of a multi-process run of the collective predict (launched by tests/test_predict_dist_gpu.py):

    RANK=r WORLD_SIZE=R MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_predict_worker.py --out DIR --mode M [...]

Every rank uses cuda:0 (CUDA IPC between processes on one GPU), plumbing over gloo.  Train batches are the CriteoSynth
batches of tests/dist_worker.py (seed 100 + rank), test batches use seed 200 + rank; initial W0 / V0 as there.

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
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WND_HIDDEN = (16,)
NFM_HIDDEN = (32, 16)
CAP_MULT = 2  # keyed capacity = CAP_MULT * F


def model_id(name):
    from lightctr_b200 import capi
    return {"ffm": capi.MODEL_FFM, "fm": capi.MODEL_FM, "nfm": capi.MODEL_NFM, "wnd": capi.MODEL_WND}[name]


def field_cnt(model):
    return 39 if model in ("ffm", "wnd") else 0


def make_params(F, k, model):
    rng = np.random.default_rng(5)
    W0 = (rng.standard_normal(F) * 0.01).astype(np.float32)
    rowlen = k * (39 if model == "ffm" else 1)
    V0 = (rng.standard_normal(F * rowlen) / np.sqrt(k)).astype(np.float32)
    return W0, V0


def train_batches(F, rows, steps, rank):
    from lightctr_b200.data import CriteoSynth
    gen = CriteoSynth(F, seed=100 + rank)
    return [gen.batch(rows) for _ in range(steps)]


def test_batches(F, rows, n, rank):
    from lightctr_b200.data import CriteoSynth
    gen = CriteoSynth(F, seed=200 + rank)
    return [gen.batch(rows) for _ in range(n)]


def make_context(model, F, k, rank, world, rows, keyed=False, hidden=None):
    """the cfg of every run here; world = 1 gives the reference context of the same cfg"""
    from lightctr_b200 import capi
    if hidden is None:
        hidden = {"wnd": WND_HIDDEN, "nfm": NFM_HIDDEN}.get(model, ())
    kw = dict(device=0, rank=rank, world=world, minibatch_size=2 * rows, max_nnz=rows * 200, hidden=hidden)
    if keyed:
        return capi.Context(model_id(model), CAP_MULT * F, k, field_cnt(model), key_mode=capi.KEYS_HASHED, **kw)
    return capi.Context(model_id(model), F, k, field_cnt(model), **kw)


def upload(ctx, model, slot, batch, keyed=False):
    from lightctr_b200 import dist as ldist
    rp, fid, fld, lab = batch
    fld = fld if field_cnt(model) else None
    if keyed:
        ctx.upload_batch_keys(slot, rp, ldist.fmix64(fid), fld, None, lab)
    else:
        ctx.upload_batch(slot, rp, fid, fld, None, lab)


def empty_batch():
    return (np.zeros(1, np.int64), np.zeros(0, np.uint32), np.zeros(0, np.uint16), np.zeros(0, np.int32))


def layer_dims(model, k):
    return [39 * k] + list(WND_HIDDEN) + [1] if model == "wnd" else [k] + list(NFM_HIDDEN) + [1]


def dense_layers(model, k):
    rng = np.random.default_rng(77)
    dims = layer_dims(model, k)
    return [((rng.random((dims[i + 1], dims[i]), dtype=np.float32) - 0.5).astype(np.float32),
             np.zeros(dims[i + 1], np.float32)) for i in range(len(dims) - 1)]


def start(args, rank, world, model=None, keyed=False):
    from lightctr_b200 import dist as ldist
    model = model or args.model
    ctx = make_context(model, args.F, args.k, rank, world, args.rows, keyed=keyed)
    if not keyed:
        ctx.upload_params(*make_params(args.F, args.k, model))
    ldist.connect(ctx)
    return ctx


def run_parity(args, rank, world, out, arrs):
    ctx = start(args, rank, world, keyed=args.keyed)
    for b in train_batches(args.F, args.rows, args.steps, rank):
        upload(ctx, args.model, 0, b, keyed=args.keyed)
        ctx.train_step(0)
    upload(ctx, args.model, 1, test_batches(args.F, args.test_rows, 1, rank)[0], keyed=args.keyed)
    arrs["pctr"] = ctx.predict(1)
    if args.keyed:  # the test upload created the rows of its unseen keys
        arrs["keys"] = ctx.download_keys()
    arrs["W"], arrs["V"] = ctx.download_params()
    return ctx


def run_interleave(args, rank, world, out, arrs):
    ctx = start(args, rank, world)
    tb = train_batches(args.F, args.rows, 3, rank)
    t1, t2 = test_batches(args.F, args.test_rows, 2, rank)
    launches = []

    def step(i):
        upload(ctx, args.model, 0, tb[i])
        n = ctx.launch_count()
        ctx.train_step(0)
        launches.append(ctx.launch_count() - n)
        arrs["W%d" % i], arrs["V%d" % i] = ctx.download_params()

    upload(ctx, args.model, 1, t1)
    upload(ctx, args.model, 2, t2)
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
    for l, (w, b) in enumerate(dense_layers("wnd", args.k)):
        ctx.mlp_upload(l, w, b)
    upload(ctx, "wnd", 0, train_batches(args.F, args.rows, 1, rank)[0])
    upload(ctx, "wnd", 1, test_batches(args.F, args.test_rows, 1, rank)[0])
    arrs["p1a"], arrs["p1b"] = ctx.predict(1), ctx.predict(1)
    out["loss"] = ctx.train_step(0)[0]
    arrs["p2"] = ctx.predict(1)
    return ctx


def run_empty(args, rank, world, out, arrs):
    from lightctr_b200 import dist as ldist
    ctx = start(args, rank, world, keyed=args.keyed)
    dense = args.model in ("nfm", "wnd")
    if dense:
        for l, (w, b) in enumerate(dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
    if args.model == "nfm":
        ldist.attach_dense_allreduce(ctx)
    predicts = args.model != "nfm"
    share = test_batches(args.F, args.test_rows, 1, rank)[0] if rank == 0 else empty_batch()
    upload(ctx, args.model, 1, share, keyed=args.keyed)
    if predicts:
        arrs["pctr"] = ctx.predict(1)
    train = train_batches(args.F, args.rows, 1, rank)[0] if rank == 0 else empty_batch()
    upload(ctx, args.model, 0, train, keyed=args.keyed)
    loss, correct = ctx.train_step(0)
    out["stats"] = [loss, correct]
    out["reduced"] = list(ldist.reduce_stats(loss, correct))
    if predicts:
        arrs["pctr_after"] = ctx.predict(1)
    if args.keyed:
        arrs["keys"] = ctx.download_keys()
    arrs["W"], arrs["V"] = ctx.download_params()
    if dense:
        dims = layer_dims(args.model, args.k)
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
    batch = test_batches(args.F, rows, 1, rank)[0] if rows else empty_batch()
    upload(ctx, args.model, 1, batch)
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
    upload(ctx, "fm", 0, train_batches(args.F, args.rows, 1, rank)[0])
    upload(ctx, "fm", 1, test_batches(args.F, args.test_rows, 1, rank)[0])
    ctx.train_step(0)
    out["quirk"] = attempt(lambda: ctx.predict(1, quirk_sumvx_slot=0))
    arrs["after_quirk"] = ctx.predict(1)  # the refusal launched nothing: the ranks still agree on the protocol
    dist.barrier()  # no peer uses this context's memory any more
    ctx.close()
    nfm = make_context("nfm", args.F, args.k, rank, world, args.rows, hidden=(16,))
    ldist.connect(nfm)
    upload(nfm, "nfm", 1, test_batches(args.F, args.test_rows, 1, rank)[0])
    out["nfm"] = attempt(lambda: nfm.predict(1))
    dist.barrier()
    nfm.close()
    # rank 0's test batch: 20000 distinct rows all owned by rank 0, more than its inbox from rank 0 holds (3 * max_nnz /
    # (2 * world) + 4096 = 19096 records with max_nnz = 20000)
    over = make_context("fm", 65536, args.k, rank, world, 100)
    over.upload_params(*make_params(65536, args.k, "fm"))
    ldist.connect(over)
    if rank == 0:
        fid = (2 * np.arange(20000)).astype(np.uint32)
        batch = (np.arange(0, 20001, 100).astype(np.int64), fid, None, np.zeros(200, np.int32))
    else:
        batch = test_batches(65536, 100, 1, rank)[0]
    upload(over, "fm", 1, batch)
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
    import torch
    import torch.distributed as dist
    torch.cuda.set_device(0)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out, arrs = {"rank": rank}, {}
    run = {"parity": run_parity, "interleave": run_interleave, "wnd": run_wnd, "empty": run_empty, "metrics": run_metrics,
           "refuse": run_refuse}[args.mode]
    ctx = run(args, rank, world, out, arrs)
    dist.barrier()
    np.savez(os.path.join(args.out, "rank%d.npz" % rank), **arrs)
    with open(os.path.join(args.out, "rank%d.json" % rank), "w") as f:
        json.dump(out, f)
    dist.barrier()
    ctx.close()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
