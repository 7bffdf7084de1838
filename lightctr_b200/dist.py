"""Process-group plumbing of the multi-GPU path (one process per GPU, torch.distributed for rendezvous only).

The data path itself is CUDA (csrc/dist.cu: unique-id pull / push over NVLink peer memory + device-side barriers);
this module only (a) exchanges the CUDA-IPC handles every rank exports, (b) reduces the per-rank step statistics,
(c) offers the shard arithmetic used on both sides of the C ABI.  Replaces the reference's master/worker
bootstrap (distribut/master.h:76-190, dist_machine_abst.h:53-87) for the single-box case.
"""
import os
import re
import struct

import numpy as np


def owner_of(fid, world):
    """Table sharding of dist.cu: row f lives on rank f % world at shard-local index f // world."""
    fid = np.asarray(fid)
    return fid % world, fid // world


def exchange_blobs(blob, group=None):
    """all-gather one bytes object per rank, returned concatenated in rank order (+ the per-rank size)."""
    import torch.distributed as dist
    world = dist.get_world_size(group)
    out = [None] * world
    dist.all_gather_object(out, blob, group=group)
    assert all(len(b) == len(blob) for b in out)
    return b"".join(out), len(blob)


def connect(ctx, group=None):
    """Export this rank's IPC handles, gather everyone's, map the peers, and barrier."""
    import torch.distributed as dist
    allb, per = exchange_blobs(ctx.ipc_export(), group)
    ctx.ipc_import(allb, per)
    dist.barrier(group)


class _DevArray:
    """Zero-copy view of a raw device pointer for torch.as_tensor (CUDA array interface v2)."""

    def __init__(self, ptr, n):
        self.__cuda_array_interface__ = {"shape": (int(n),), "typestr": "<f4", "data": (int(ptr), False), "version": 2}


def attach_dense_allreduce(ctx, group=None):
    """Install the dense-gradient all-reduce of the data-parallel NFM layers (lctr_set_dense_allreduce): NCCL on the
    context's own stream (replaces Worker_RingReduce::syncGradient, distribut/ring_collect.h:48-72).  With a gloo group
    (tests: several ranks sharing one GPU) the sum goes through the host."""
    import torch
    import torch.distributed as dist

    def fn(ptr, n, stream):
        t = torch.as_tensor(_DevArray(ptr, n), device="cuda")
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            if dist.get_backend(group) == "nccl":
                dist.all_reduce(t, group=group)
            else:
                h = t.cpu()
                dist.all_reduce(h, group=group)
                t.copy_(h)
    ctx.set_dense_allreduce(fn)


def reduce_stats(loss, correct, group=None):
    """Sum of the per-rank (summed logloss, correct count): what a single process would print for the global batch."""
    import torch
    import torch.distributed as dist
    t = torch.tensor([loss, correct], dtype=torch.float64)
    if dist.get_backend(group) == "nccl":
        t = t.cuda()
    dist.all_reduce(t, group=group)
    return float(t[0]), float(t[1])


def eval_global(ctx, slot, labels, group=None, weights=None):
    """(summed logloss, correct count, AUC) of the whole test set a sharded trainer just predicted (lctr_predict on `slot`,
    collective): every rank passes the labels of its own rows.  This rank's pCTR is downloaded, (pCTR, labels) are
    all-gathered in rank order and the concatenation is evaluated on every rank (lctr_eval_pred), so every rank returns the
    same numbers, equal bit for bit to lctr_eval on one GPU holding the concatenated batch (rank 0's rows first) with the
    same pCTR.  Shares may be uneven, or empty.  Host traffic per rank: R * n * 8 B, with n the largest share.
    weights (one per row of this rank, every rank passing them or none): (pCTR, label, weight) are gathered alike and the
    weighted metrics of lctr_eval_pred_weighted are returned, equal bit for bit to that call on the concatenation."""
    import torch.distributed as dist
    y = np.ascontiguousarray(labels, np.int32)
    w = None if weights is None else np.ascontiguousarray(weights, np.float32)
    p = ctx.download_pred(slot)
    world = dist.get_world_size(group)
    # every rank's row, label and weight counts first: a mismatch on any rank fails the call on every rank, none is left
    # waiting
    mine = [len(p), len(y)] + ([] if w is None else [len(w)])
    counts = np.frombuffer(exchange_blobs(np.array(mine, np.int64).tobytes(), group)[0], np.int64).reshape(world, len(mine))
    bad = [r for r in range(world) if (counts[r] != counts[r, 0]).any()]
    if bad:
        what = "labels" if w is None else "labels or weights"
        raise ValueError("eval_global: slot %d: pCTR rows and %s differ on rank(s) %s (%s)" %
                         (slot, what, bad, ", ".join(" vs ".join("%d" % v for v in counts[r]) for r in bad)))
    counts = counts[:, 0]
    n_max = int(counts.max())
    cols = 2 if w is None else 3
    blob = np.zeros(cols * n_max, np.float32)
    blob[:len(p)] = p
    blob.view(np.int32)[n_max:n_max + len(y)] = y
    if w is not None:
        blob[2 * n_max:2 * n_max + len(w)] = w
    allb, per = exchange_blobs(blob.tobytes(), group)
    parts = [np.frombuffer(allb[r * per:(r + 1) * per], np.float32) for r in range(world)]
    pctr = np.concatenate([b[:counts[r]] for r, b in enumerate(parts)])
    lab = np.concatenate([b.view(np.int32)[n_max:n_max + counts[r]] for r, b in enumerate(parts)])
    if w is None:
        return ctx.eval_pred(pctr, lab)
    wts = np.concatenate([b[2 * n_max:2 * n_max + counts[r]] for r, b in enumerate(parts)])
    return ctx.eval_pred(pctr, lab, wts)


def merge_shards(parts, world, n_rows):
    """Combine per-rank full-size arrays whose only valid rows are the owned ones (lctr_download_params, world > 1)."""
    rowlen = len(parts[0]) // n_rows
    out = np.zeros_like(parts[0]).reshape(n_rows, rowlen)
    for r, p in enumerate(parts):
        out[r::world] = p.reshape(n_rows, rowlen)[r::world]
    return out.reshape(-1)


def fmix64(x):
    """MurmurHash3's 64-bit finaliser, mod 2^64 (csrc/keys.cuh: fmix64)."""
    k = np.array(x, dtype=np.uint64, copy=True)
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xff51afd7ed558ccd)
        k ^= k >> np.uint64(33)
        k *= np.uint64(0xc4ceb9fe1a85ec53)
        k ^= k >> np.uint64(33)
    return k


def owner_of_key(keys, world):
    """Rank that owns each hashed key of a keyed context on `world` (a power of two) ranks: the top log2(world) bits of
    fmix64(key) (csrc/keys.cuh: owner_of_key).  Its row l there is global row l * world + rank."""
    assert world >= 1 and world & (world - 1) == 0, world
    shift = world.bit_length() - 1
    if shift == 0:
        return np.zeros(np.shape(keys), np.int64)
    return (fmix64(keys) >> np.uint64(64 - shift)).astype(np.int64)


def merge_keyed_shards(keys, W, V, world):
    """key -> (W, V row) of a sharded keyed table.  keys[r] is rank r's download_keys() (its local rows in order), W[r] /
    V[r] its download_params() arrays, in which local row l sits at global row l * world + r."""
    out = {}
    for r in range(world):
        kr = np.asarray(keys[r], np.uint64)
        g = np.arange(len(kr), dtype=np.int64) * world + r
        rowlen = len(V[r]) // len(W[r])
        Vr = np.asarray(V[r]).reshape(-1, rowlen)
        for key, w, v in zip(kr.tolist(), np.asarray(W[r])[g], Vr[g]):
            assert key not in out, "key %d held by more than one rank" % key
            out[key] = (w, v)
    return out


# ---- checkpoints of sharded trainers (lctr_save_checkpoint per rank, lctr_load_checkpoint[_shards]) --------------------
_SHARD_NAME = re.compile(r"\.rank(\d+)-of-(\d+)$")


def shard_path(prefix, rank, world):
    """File of rank `rank` in a save of a world-`world` run under `prefix`."""
    return "%s.rank%d-of-%d" % (prefix, rank, world)


def delta_path(prefix, seq, rank=0, world=1):
    """File of the seq-th incremental save (lctr_save_checkpoint_delta) of rank `rank` of a world-`world` run under
    `prefix`: shard_path's name with ".delta<seq>" after it, so find_shards never takes it for a full save."""
    return "%s.delta%d" % (shard_path(prefix, rank, world), seq)


def checkpoint_info(path):
    """(step, adam_iter, world, rank) from the header of a checkpoint file (csrc/checkpoint.cu: CkptHeader, CkptShard),
    full or incremental; a single-GPU full file reads as world 1, rank 0."""
    with open(path, "rb") as f:
        head = f.read(136 + 24)
    if len(head) < 136 or head[:8] not in (b"LCTRCKP1", b"LCTRCKS1", b"LCTRCKD1"):
        raise ValueError("%s is not a lightctr_b200 checkpoint" % path)
    adam_iter, step = struct.unpack_from("<QQ", head, 48)
    if head[:8] == b"LCTRCKP1":
        return step, adam_iter, 1, 0
    if len(head) < 160:
        raise ValueError("%s: short shard header" % path)
    world, rank = struct.unpack_from("<ii", head, 136)
    return step, adam_iter, world, rank


def find_shards(prefix):
    """The files of the save under `prefix`, in rank order: every `prefix.rank<r>-of-<R>` beside it.  Refuses files of
    two different worlds, a rank given twice, and a set with gaps."""
    d, base = os.path.split(prefix)
    found = {}
    for name in os.listdir(d or "."):
        if not name.startswith(base + ".rank"):
            continue
        m = _SHARD_NAME.search(name[len(base):])
        if not m or m.start() != 0:
            continue
        r, w = int(m.group(1)), int(m.group(2))
        if (r, w) in found:
            raise ValueError("rank %d of world %d appears twice under %s: %s, %s" % (r, w, prefix, found[(r, w)], name))
        found[(r, w)] = name
    if not found:
        raise FileNotFoundError("no checkpoint files %s.rank<r>-of-<R>" % prefix)
    worlds = sorted({w for _, w in found})
    if len(worlds) > 1:
        raise ValueError("files of several saves under %s (worlds %s)" % (prefix, worlds))
    world = worlds[0]
    missing = [r for r in range(world) if (r, world) not in found]
    if missing or len(found) != world:
        raise ValueError("incomplete save under %s: world %d, ranks %s missing" % (prefix, world, missing))
    return [os.path.join(d, found[(r, world)]) for r in range(world)], world


def save_sharded(ctx, prefix, group=None):
    """Every rank writes its shard to shard_path(prefix, rank, world); the ranks then barrier and check that they all
    saved the same step."""
    rank, world = ctx.cfg.rank, ctx.cfg.world
    path = shard_path(prefix, rank, world)
    ctx.save_checkpoint(path)
    if world > 1:
        import torch.distributed as dist
        dist.barrier(group)
        steps = [None] * world
        dist.all_gather_object(steps, checkpoint_info(path)[:2], group=group)
        if any(s != steps[0] for s in steps):
            raise RuntimeError("save_sharded: the ranks saved different (step, adam_iter): %s" % steps)
    return path


def load_sharded(ctx, prefix, group=None):
    """Load the save under `prefix` into this rank's context, whatever world wrote it: the rank's own file when the world
    is unchanged, else every file, each rank taking the rows it owns (lctr_load_checkpoint_shards).  Returns the world
    of the save."""
    paths, world = find_shards(prefix)
    if world == ctx.cfg.world:
        ctx.load_checkpoint(paths[ctx.cfg.rank])
    else:
        ctx.load_checkpoint_shards(paths)
    if ctx.cfg.world > 1:  # nobody starts a collective upload while a peer is still reading
        import torch.distributed as dist
        dist.barrier(group)
    return world
