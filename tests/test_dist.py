"""Multi-GPU path (SURVEY.md 8e): owner-sharded tables, per-batch unique-id pull / push, owner-side update.

CPU (gloo, world_size 2): the process-group plumbing and an emulation of the exchange protocol with the oracle's
arithmetic must equal the single-process oracle step on the concatenated global batch.
GPU (-m gpu): the CUDA implementation, 2 ranks (both on cuda:0 over CUDA IPC), against the same oracle."""
import numpy as np
import pytest

import multirank as mr


def _oracle_global(oracle_api, world, F, k, rows, steps, model="fm"):
    per_rank = [mr.train_batches(F, rows, steps, r) for r in range(world)]
    W, V = mr.make_params(F, k, model)
    Fc = 39 if model == "ffm" else 0
    accum = np.zeros(F * (k * max(Fc, 1) + 1), np.float32)
    stats = []
    for s in range(steps):
        rp, fid, fld, lab = mr.global_batch([b[s] for b in per_rank])
        ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, Fc)
        if model == "ffm":
            o = oracle_api.FFMOracle(ds, k, W, V)
            o.s1[:] = accum
            loss, acc = o.epoch()
            W, V, accum = o.W.copy(), o.V.copy(), o.s1.copy()
        else:
            o = oracle_api.FMOracle(ds, k, W, V)
            o.accum[:] = accum
            loss, acc = o.epoch()
            W, V, accum = o.W.copy(), o.V.copy(), o.accum.copy()
        stats.append((loss, acc * ds.rows))
    return W, V, stats


def _oracle_global_nfm(oracle_api, world, F, k, rows, steps):
    """Single-process NFM oracle on the concatenated global batch: one minibatch of world*rows samples per step, masks
    all ones, the same initial dense layers as the ranks."""
    per_rank = [mr.train_batches(F, rows, steps, r) for r in range(world)]
    W, V = mr.make_params(F, k, "nfm")
    accum = np.zeros(F * (k + 1), np.float32)
    mlp0 = mr.dense_layers("nfm", k)
    nl = len(mlp0)
    state = {"weight": [w.reshape(-1).copy() for w, _ in mlp0], "bias": [b.copy() for _, b in mlp0], "accum": None}
    stats = []
    for s in range(steps):
        rp, fid, fld, lab = mr.global_batch([b[s] for b in per_rank])
        ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, 0)
        B = world * rows
        o = oracle_api.NFMOracle(ds, k, list(mr.NFM_HIDDEN), W=W, V=V, batch_size=B, minibatch=B)
        o.accum[:] = accum
        for l in range(nl):
            o.mlp.arrays("weight", l)[:] = state["weight"][l]
            o.mlp.arrays("bias", l)[:] = state["bias"][l]
            o.mlp.arrays("mask", l)[:] = 1.0
            if state["accum"] is not None:
                o.mlp.arrays("accum", l)[:] = state["accum"][l]
        loss, acc = o.epoch()
        W, V, accum = o.W.copy(), o.V.copy(), o.accum.copy()
        state = {k2: [o.mlp.arrays(k2, l).copy() for l in range(nl)] for k2 in ("weight", "bias", "accum")}
        stats.append((loss, acc * ds.rows))
    return W, V, stats, state


def _check(out, world, F, k, oracle, tol):
    from lightctr_b200 import dist as ldist
    parts = mr.load(out, world)
    W = ldist.merge_shards([p["W"] for p in parts], world, F)
    V = ldist.merge_shards([p["V"] for p in parts], world, F)
    Wo, Vo, so = oracle
    for (lg, cg), (lo, co) in zip(parts[0]["stats"], so):
        assert abs(lg - lo) <= 1e-5 * abs(lo) and cg == co
    assert np.max(np.abs(W - Wo)) < tol and np.max(np.abs(V - Vo)) < tol


def test_shard_arithmetic():
    from lightctr_b200 import dist as ldist
    f = np.arange(37)
    o, l = ldist.owner_of(f, 4)
    assert np.array_equal(o, f % 4) and np.array_equal(l, f // 4)
    parts = []
    full = np.arange(12 * 3, dtype=np.float32)
    for r in range(4):
        p = np.zeros_like(full).reshape(12, 3)
        p[r::4] = full.reshape(12, 3)[r::4]
        parts.append(p.reshape(-1))
    assert np.array_equal(ldist.merge_shards(parts, 4, 12), full)


def test_protocol_emulation_gloo_world2(oracle_api, tmp_path):
    """world_size-2 gloo run of the pull / push / owner-update protocol == single-process oracle on the global batch."""
    F, k, rows, steps = 5000, 8, 64, 3
    mr.launch("dist_worker.py", tmp_path, ["--mode", "emu", "--F", str(F), "--k", str(k), "--rows", str(rows), "--steps",
                                           str(steps)], timeout=600)
    _check(tmp_path, 2, F, k, _oracle_global(oracle_api, 2, F, k, rows, steps), 2e-6)


@pytest.mark.gpu
def test_cuda_two_ranks_one_device(oracle_api, tmp_path):
    """The CUDA multi-GPU path with 2 ranks sharing cuda:0 (CUDA IPC between processes), vs the oracle."""
    F, k, rows, steps = 20000, 16, 256, 3
    mr.launch("dist_worker.py", tmp_path, ["--mode", "gpu", "--same-device", "--F", str(F), "--k", str(k), "--rows",
                                           str(rows), "--steps", str(steps)])
    _check(tmp_path, 2, F, k, _oracle_global(oracle_api, 2, F, k, rows, steps), 2e-5)


@pytest.mark.gpu
def test_cuda_two_ranks_ffm(oracle_api, tmp_path):
    """FFM (39 fields, k=4) over 2 ranks: rows of Fc*k floats travel through the same pull / push kernels."""
    F, k, rows, steps = 6000, 4, 128, 2
    mr.launch("dist_worker.py", tmp_path, ["--mode", "gpu", "--same-device", "--model", "ffm", "--F", str(F), "--k",
                                           str(k), "--rows", str(rows), "--steps", str(steps)])
    _check(tmp_path, 2, F, k, _oracle_global(oracle_api, 2, F, k, rows, steps, model="ffm"), 5e-5)


@pytest.mark.gpu
def test_cuda_two_ranks_nfm(oracle_api, tmp_path):
    """NFM over 2 ranks: embeddings owner-sharded (pull / push), dense layers replicated with the per-rank dW / db summed
    through lctr_set_dense_allreduce before the dense Adagrad (gloo through the host here: both ranks share cuda:0)."""
    F, k, rows, steps = 8000, 16, 128, 3
    mr.launch("dist_worker.py", tmp_path, ["--mode", "gpu", "--same-device", "--model", "nfm", "--F", str(F), "--k",
                                           str(k), "--rows", str(rows), "--steps", str(steps)])
    Wo, Vo, so, mlp = _oracle_global_nfm(oracle_api, 2, F, k, rows, steps)
    _check(tmp_path, 2, F, k, (Wo, Vo, so), 5e-5)
    parts = mr.load(tmp_path)
    for l in range(len(mlp["weight"])):
        for r in range(2):  # replicas stay identical and equal to the oracle's layers
            assert np.max(np.abs(parts[r]["mlp_w%d" % l] - mlp["weight"][l])) < 5e-5
            assert np.max(np.abs(parts[r]["mlp_b%d" % l] - mlp["bias"][l])) < 5e-5
        assert np.array_equal(parts[0]["mlp_w%d" % l], parts[1]["mlp_w%d" % l])
