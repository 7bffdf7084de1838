"""Process-group plumbing of the multi-GPU path (one process per GPU, torch.distributed for rendezvous only).

The data path itself is CUDA (csrc/dist.cu: unique-id pull / push over NVLink peer memory + device-side barriers);
this module only (a) exchanges the CUDA-IPC handles every rank exports, (b) reduces the per-rank step statistics,
(c) offers the shard arithmetic used on both sides of the C ABI.  Replaces the reference's master/worker
bootstrap (distribut/master.h:76-190, dist_machine_abst.h:53-87) for the single-box case.
"""
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
