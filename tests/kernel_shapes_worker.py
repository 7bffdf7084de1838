"""Batches and runs of tests/test_kernel_shapes_gpu.py.  Some kernel choices are read from the environment once per process
(LCTR_FWD_COALESCED, LCTR_FFM_WARP), so a run under another setting happens in a process of its own:

    LCTR_FWD_COALESCED=0 python tests/kernel_shapes_worker.py IN.npz OUT.npz

IN.npz: model, k, Fc, det, lr, the batch (rp, fid, fld, val -- empty = no values --, lab) and states W<i>, V<i>, S<i>
(S = updater state s1); optional opt (updater, default Adagrad), l2 (default 0.001) and mb (minibatch_size, default 0 =
the rows of the step).  For each state: upload it, then a train step (train = 1: loss<i>, cnt<i>, Wout<i>, Vout<i> and the
step's pCTR pred<i>) or a predict (train = 0: pctr<i>, and sumvx<i> for FM).  OUT.npz holds the results."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def make_batch(seed, F=4000, rows=300, Fc=0, with_val=True):
    """rows of 0, 1, 63, 64, 65 (the forward's 64-feature passes), 129 (past the order-free kernel's 128-entry window at
    k = 16) and 300 entries, the rest 2..40; ids 0..2 shared by most rows; values in [0.25, 1.75) or absent; fields
    unordered within a row.  Returns rp, fid, fld (uint16), val (None when absent), lab."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 41, rows)
    special = (0, 1, 63, 64, 65, 129, 300)
    lens[np.arange(len(special)) * (rows // len(special))] = special
    fid = []
    for r, n in enumerate(lens):
        ids = rng.choice(np.arange(3, F), n, replace=False)
        if n >= 3:
            ids[int(rng.integers(0, n))] = r % 3
        fid.append(ids)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fid = np.concatenate(fid).astype(np.uint32)
    fld = rng.integers(0, max(Fc, 1), len(fid)).astype(np.uint16)
    val = (0.25 + 1.5 * rng.random(len(fid))).astype(np.float32) if with_val else None
    lab = (rng.random(rows) < 0.4).astype(np.int32)
    return rp, fid, fld, val, lab


def make_params(seed, F, k, Fc=0):
    rng = np.random.default_rng(seed + 1000)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    scale = 0.1 / np.sqrt(k) if Fc == 0 else 0.1
    V = (rng.standard_normal(F * k * max(Fc, 1)) * scale).astype(np.float32)
    return W, V


def run(inp):
    from lightctr_b200 import capi
    model, k, Fc, det = int(inp["model"]), int(inp["k"]), int(inp["Fc"]), int(inp["det"])
    rp, fid, fld, lab = inp["rp"], inp["fid"], inp["fld"], inp["lab"]
    val = inp["val"] if len(inp["val"]) else None
    F = len(inp["W0"])
    opt = int(inp["opt"]) if "opt" in inp else capi.OPT_ADAGRAD
    l2 = float(inp["l2"]) if "l2" in inp else 0.001
    mb = int(inp["mb"]) if "mb" in inp else 0
    ctx = capi.Context(model, F, k, Fc, deterministic=det, lr=float(inp["lr"]), optimizer=opt, l2=l2, minibatch_size=mb)
    ctx.upload_batch(0, rp, fid, fld if Fc else None, val, lab)
    out = {}
    i = 0
    while f"W{i}" in inp:
        ctx.upload_params(inp[f"W{i}"], inp[f"V{i}"])
        if f"S{i}" in inp:
            ctx.upload_opt_state(inp[f"S{i}"])
        if int(inp["train"]):
            out[f"loss{i}"], out[f"cnt{i}"] = ctx.train_step(0)
            out[f"Wout{i}"], out[f"Vout{i}"] = ctx.download_params()
            out[f"pred{i}"] = ctx.download_pred(0)
        else:
            out[f"pctr{i}"] = ctx.predict(0)
            if model == capi.MODEL_FM:
                out[f"sumvx{i}"] = ctx.download_sumvx(0)
        i += 1
    ctx.close()
    return out


if __name__ == "__main__":
    with np.load(sys.argv[1]) as z:
        inp = {n: z[n] for n in z.files}
    np.savez(sys.argv[2], **run(inp))
