"""One rank of a multi-process run of the multi-GPU path (launched by tests/test_dist.py and usable by hand):

    RANK=r WORLD_SIZE=R MASTER_ADDR=127.0.0.1 MASTER_PORT=p python tests/dist_worker.py --out DIR [...]

mode=gpu   : the real CUDA path (csrc/dist.cu); with --same-device every rank uses cuda:0 (IPC between processes on
             one GPU -- slow barriers, but exercises every kernel), plumbing over gloo.  --probe: the updater is a unit
             SGD step (OPT_PS_SGD with lr = the global batch, so w1 = w0 - g) and each step's pCTR is saved as well.
mode=emu   : CPU emulation of the same protocol with the oracle's arithmetic and gloo collectives (pull = all ranks
             read the owner's rows, push = all_to_all of (fid, grad row) records, owner merges + applies): checks that
             the protocol is the single-process step, on machines without a GPU."""
import argparse

import numpy as np

import multirank as mr


def run_gpu(args, rank, world):
    import torch
    import torch.distributed as dist
    from lightctr_b200 import capi, dist as ldist
    batches, (W0, V0) = mr.train_batches(args.F, args.rows, args.steps, rank), mr.make_params(args.F, args.k, args.model)
    dev = 0 if args.same_device else rank
    torch.cuda.set_device(dev)
    ctx = mr.make_context(args.model, args.F, args.k, rank, world, minibatch_size=world * args.rows,
                          max_nnz=args.rows * 200, device=dev,
                          **(dict(optimizer=capi.OPT_PS_SGD, lr=float(world * args.rows)) if args.probe else {}))
    ctx.upload_params(W0, V0)
    ldist.connect(ctx)
    if args.model in ("nfm", "wnd"):
        for l, (w, b) in enumerate(mr.dense_layers(args.model, args.k)):
            ctx.mlp_upload(l, w, b)
    if args.model == "nfm":  # Wide&Deep without the hook: every rank trains its own dense layers
        ldist.attach_dense_allreduce(ctx)
    stats, preds = [], []
    for b in batches:
        mr.upload(ctx, args.model, 0, b)
        l, c = ctx.train_step(0)
        stats.append(ldist.reduce_stats(l, c))
        if args.probe:
            preds.append(ctx.download_pred(0))
    dist.barrier()
    W, V = ctx.download_params()
    arrs = {"W": W, "V": V, "stats": np.array(stats)}
    if args.probe:
        arrs["pred"] = np.concatenate(preds)
    dims = mr.layer_dims(args.model, args.k)
    for l in range(len(dims) - 1):
        arrs["mlp_w%d" % l], arrs["mlp_b%d" % l] = ctx.mlp_download(l, dims[l], dims[l + 1])
    mr.save(args.out, rank, arrs)
    dist.barrier()
    ctx.close()


def run_emu(args, rank, world):
    import torch
    import torch.distributed as dist
    from oracle import api
    batches, (W0, V0) = mr.train_batches(args.F, args.rows, args.steps, rank), mr.make_params(args.F, args.k, args.model)
    F, k = args.F, args.k
    mine = np.arange(rank, F, world)
    W, V = W0[mine].copy(), V0.reshape(F, k)[mine].copy()          # my shard
    acc = np.zeros((len(mine), k + 1), np.float32)                   # adagrad accum of my shard: [:,0]=W, [:,1:]=V
    stats = []
    for rp, fid, fld, lab in batches:
        uniq = np.unique(fid)                                        # pull_map keys (distributed_algo_abst.h:181-190)
        # pull: every rank serves the rows it owns (all_gather of shards == what peer loads read)
        shards_W, shards_V = [None] * world, [None] * world
        dist.all_gather_object(shards_W, W)
        dist.all_gather_object(shards_V, V)
        cW, cV = np.zeros(F, np.float32), np.zeros((F, k), np.float32)
        for r in range(world):
            cW[r::world], cV[r::world] = shards_W[r], shards_V[r]
        ds = api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, 0)
        o = api.FMOracle(ds, k, cW, cV.reshape(-1))
        loss, accu = o.forward_backward()                            # local update_g
        gW, gV = o.update_g[:F], o.update_g[F:].reshape(F, k)
        # push: records to owners
        send = [None] * world
        for r in range(world):
            sel = uniq[uniq % world == r]
            send[r] = (sel, gW[sel].copy(), gV[sel].copy())
        recv = [None] * world
        dist.all_to_all_object = None
        gathered = [None] * world
        dist.all_gather_object(gathered, send)
        recv = [gathered[src][rank] for src in range(world)]
        # owner: merge in source order, then Adagrad with the GLOBAL minibatch size
        g = np.zeros((len(mine), k + 1), np.float32)
        for sel, gw, gv in recv:
            l = sel // world
            np.add.at(g[:, 0], l, gw)
            np.add.at(g[:, 1:], l, gv)
        B = world * args.rows
        L = api.lib()
        wv = np.concatenate([W[:, None], V], axis=1).reshape(-1).copy()
        gg, aa = g.reshape(-1).copy(), acc.reshape(-1).copy()
        L.orc_adagrad(len(wv), wv, gg, aa, B, np.float32(0.05))
        wv = wv.reshape(len(mine), k + 1)
        W, V, acc = wv[:, 0].copy(), wv[:, 1:].copy(), aa.reshape(len(mine), k + 1)
        t = torch.tensor([loss, accu * len(lab)], dtype=torch.float64)
        dist.all_reduce(t)
        stats.append((float(t[0]), float(t[1])))
    Wf, Vf = np.zeros(F, np.float32), np.zeros((F, k), np.float32)
    Wf[mine], Vf[mine] = W, V
    mr.save(args.out, rank, {"W": Wf, "V": Vf.reshape(-1), "stats": np.array(stats)})
    dist.barrier()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--mode", default="gpu")
    ap.add_argument("--model", default="fm")
    ap.add_argument("--F", type=int, default=20000)
    ap.add_argument("--k", type=int, default=16)
    ap.add_argument("--rows", type=int, default=256)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--out", required=True)
    ap.add_argument("--same-device", action="store_true")
    ap.add_argument("--probe", action="store_true")
    ap.add_argument("--backend", default="gloo")
    args = ap.parse_args()
    run = run_gpu if args.mode == "gpu" else run_emu
    mr.main(lambda rank, world: run(args, rank, world), backend=args.backend)


if __name__ == "__main__":
    main()
