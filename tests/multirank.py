"""Multi-rank runs of the tests: the launcher on the host side, and the problem every rank builds on the rank side.

Host side: `run` starts one process per rank and waits for all of them together, `launch` runs one of the tests/dist_*
workers that way, `load` / `load_json` read back what each rank wrote with `save`, and `global_batch` joins the ranks'
batches into the one batch a world-1 reference trains on.

Rank side: the workers and the world-1 references build their contexts, batches, parameters and dense layers from the
same functions here, so a parity test compares runs of one configuration.  Workers run as scripts from tests/, so the
repository root goes on the path here."""
import json
import os
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


# ------------------------------------------------------------------------------------------------------------------------
# host side
# ------------------------------------------------------------------------------------------------------------------------
def free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def run(world, argv, env=None, timeout=900):
    """Start `world` processes, rank r with argv(r) and os.environ plus env(r) (by default torch.distributed's variables
    on a free port), and wait for them together.  As soon as one exits non-zero, or `timeout` seconds pass, every rank
    still alive is killed and reaped, and the run fails with each rank's exit code and output: a rank blocked in a
    collective with a failed peer would otherwise hold the test until the timeout, and outlive it.
    Returns each rank's output."""
    if env is None:
        port = free_port()

        def env(r):
            return dict(RANK=str(r), WORLD_SIZE=str(world), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port),
                        LOCAL_RANK=str(r))
    logs = [tempfile.TemporaryFile("w+") for _ in range(world)]  # files, not pipes: a full pipe would block its rank
    procs, timed_out = [], False
    try:
        for r in range(world):
            procs.append(subprocess.Popen(argv(r), env=dict(os.environ, **env(r)), stdout=logs[r],
                                          stderr=subprocess.STDOUT))
        deadline = time.monotonic() + timeout
        while True:
            codes = [p.poll() for p in procs]
            if any(codes) or None not in codes:
                break
            if time.monotonic() > deadline:
                timed_out = True
                break
            time.sleep(0.1)
    finally:
        for p in procs:
            if p.poll() is None:
                p.kill()
            p.wait()
        out = []
        for f in logs:
            f.seek(0)
            out.append(f.read())
            f.close()
    codes = [p.returncode for p in procs]
    if any(codes):
        raise AssertionError("%s; exit codes %s\n%s" % (
            "timed out after %g s" % timeout if timed_out else "a rank failed", codes,
            "\n".join("--- rank %d, exit code %s ---\n%s" % (r, c, o) for r, (c, o) in enumerate(zip(codes, out)))))
    return out


def launch(worker, out, args, world=2, timeout=900):
    """tests/<worker> on `world` gloo ranks, writing under `out`"""
    os.makedirs(out, exist_ok=True)
    return run(world, lambda r: [sys.executable, os.path.join(HERE, worker), "--out", str(out)] + list(args),
               timeout=timeout)


def _path(out, rank, ext):
    return os.path.join(out, "rank%d.%s" % (rank, ext))


def save(out, rank, arrays=None, messages=None):
    """a rank's arrays into rank<r>.npz, its messages into rank<r>.json"""
    if arrays is not None:
        np.savez(_path(out, rank, "npz"), **arrays)
    if messages is not None:
        with open(_path(out, rank, "json"), "w") as f:
            json.dump(messages, f)


def load(out, world=2):
    return [dict(np.load(_path(out, r, "npz"))) for r in range(world)]


def load_json(out, world=2):
    res = []
    for r in range(world):
        with open(_path(out, r, "json")) as f:
            res.append(json.load(f))
    return res


def global_batch(batches):
    """(row_ptr, fid, field, label) batches of the ranks joined in rank order into one CSR batch"""
    rp, off = [np.zeros(1, np.int64)], 0
    for b in batches:
        rp.append(b[0][1:] + off)
        off += b[0][-1]
    return (np.concatenate(rp),) + tuple(np.concatenate([b[i] for b in batches]) for i in (1, 2, 3))


# ------------------------------------------------------------------------------------------------------------------------
# rank side
# ------------------------------------------------------------------------------------------------------------------------
NFM_HIDDEN = (32, 16)
WND_HIDDEN = (16,)
CAP_MULT = 2  # keyed capacity = CAP_MULT * F: every key a run can meet fits each owner's shard


def model_id(model):
    from lightctr_b200 import capi
    return {"ffm": capi.MODEL_FFM, "fm": capi.MODEL_FM, "nfm": capi.MODEL_NFM, "wnd": capi.MODEL_WND}[model]


def field_cnt(model):
    return 39 if model in ("ffm", "wnd") else 0


def layer_dims(model, k):
    """widths of the dense layers, [] for the models without them"""
    if model == "nfm":
        return [k] + list(NFM_HIDDEN) + [1]
    if model == "wnd":
        return [39 * k] + list(WND_HIDDEN) + [1]
    return []


def dense_layers(model, k):
    """initial (weight, bias) of each dense layer, the same on every rank"""
    rng = np.random.default_rng(77)
    dims = layer_dims(model, k)
    return [((rng.random((dims[i + 1], dims[i]), dtype=np.float32) - 0.5).astype(np.float32),
             np.zeros(dims[i + 1], np.float32)) for i in range(len(dims) - 1)]


def make_params(F, k, model):
    """initial W / V, the same on every rank"""
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


def make_context(model, F, k, rank, world, *, minibatch_size, max_nnz, keyed=False, cap=None, device=0, **kw):
    """the context of a rank (world = 1: of a reference); keyed contexts hold `cap` rows, CAP_MULT * F by default"""
    from lightctr_b200 import capi
    kw.setdefault("hidden", {"nfm": NFM_HIDDEN, "wnd": WND_HIDDEN}.get(model, ()))
    if keyed:
        F = cap or CAP_MULT * F
        kw["key_mode"] = capi.KEYS_HASHED
    return capi.Context(model_id(model), F, k, field_cnt(model), device=device, rank=rank, world=world,
                        minibatch_size=minibatch_size, max_nnz=max_nnz, **kw)


def upload(ctx, model, slot, batch, keyed=False):
    """a (row_ptr, fid, field, label) batch into `slot`; keyed: key = fmix64(fid)"""
    from lightctr_b200 import dist as ldist
    rp, fid, fld, lab = batch
    fld = fld if field_cnt(model) else None
    if keyed:
        ctx.upload_batch_keys(slot, rp, ldist.fmix64(fid), fld, None, lab)
    else:
        ctx.upload_batch(slot, rp, fid, fld, None, lab)


def main(body, backend="gloo", device=None):
    """one rank: join the process group of RANK / WORLD_SIZE (MASTER_ADDR / MASTER_PORT), body(rank, world), leave it"""
    import torch
    import torch.distributed as dist
    if device is not None:
        torch.cuda.set_device(device)
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dist.init_process_group(backend, rank=rank, world_size=world)
    body(rank, world)
    dist.destroy_process_group()
