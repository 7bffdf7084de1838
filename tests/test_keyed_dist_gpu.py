"""Keyed mode on several GPUs (csrc/dist.cu, keyed upload): 2 ranks sharing cuda:0 over CUDA IPC against a single-GPU
keyed context trained on the concatenated global batch.  Lazy init depends on (seed, key, element) only, so both start
from the same values and every key's W and V must agree after training; each key must live on its owner only."""
import numpy as np
import pytest

import multirank as mr

pytestmark = pytest.mark.gpu


def _single_gpu(model, F, k, rows, steps, seeded, world=2):
    """one keyed context on the global batch (every rank's rows, rank order), same capacity and lazy init"""
    from lightctr_b200 import dist as ldist
    per_rank = [mr.train_batches(F, rows, steps, r) for r in range(world)]
    ctx = mr.make_context(model, F, k, 0, 1, minibatch_size=world * rows, max_nnz=world * rows * 200, keyed=True)
    if seeded:
        ctx.upload_keyed_params(ldist.fmix64(np.arange(F)), *mr.make_params(F, k, model))
    for l, (w, b) in enumerate(mr.dense_layers(model, k)):
        ctx.mlp_upload(l, w, b)
    stats, seen = [], set()
    for s in range(steps):
        batch = mr.global_batch([b[s] for b in per_rank])
        seen.update(ldist.fmix64(batch[1]).tolist())
        mr.upload(ctx, model, 0, batch, keyed=True)
        stats.append(ctx.train_step(0))
    kk = ctx.download_keys()
    W, V = ctx.download_params()
    rowlen = len(V) // len(W)
    ref = {key: (W[i], V[i * rowlen:(i + 1) * rowlen]) for i, key in enumerate(kk.tolist())}
    ctx.close()
    return ref, stats, seen


def _check_train(tmp_path, model, F, k, rows, steps, tol, seeded=False):
    from lightctr_b200 import dist as ldist
    extra = ["--model", model, "--F", str(F), "--k", str(k), "--rows", str(rows), "--steps", str(steps)]
    mr.launch("dist_keyed_worker.py", tmp_path, extra + (["--seeded"] if seeded else []))
    parts = mr.load(tmp_path)
    got = ldist.merge_keyed_shards([p["keys"] for p in parts], [p["W"] for p in parts], [p["V"] for p in parts], 2)
    ref, stats, seen = _single_gpu(model, F, k, rows, steps, seeded)
    for (lg, cg), (lo, co) in zip(parts[0]["stats"], stats):
        assert abs(lg - lo) <= 1e-5 * abs(lo) and cg == co, (lg, lo, cg, co)
    assert set(got) == set(ref)
    dw = max(abs(float(got[key][0]) - float(ref[key][0])) for key in ref)
    dv = max(float(np.max(np.abs(got[key][1] - ref[key][1]))) for key in ref)
    assert dw < tol and dv < tol, (dw, dv)
    return parts, seen


def test_keyed_fm_two_ranks_lazy_init(tmp_path):
    """FM k=16 Adagrad with lazily created rows, 3 steps; placement: every key on its owner only, rows [0, n_r) there"""
    from lightctr_b200 import dist as ldist
    parts, seen = _check_train(tmp_path, "fm", 20000, 16, 256, 3, 2e-5)
    union = set()
    for r, p in enumerate(parts):
        keys = p["keys"]
        assert len(keys) > 0 and np.all(ldist.owner_of_key(keys, 2) == r)
        assert np.array_equal(p["rows"], np.arange(len(keys), dtype=np.int64) * 2 + r)
        assert union.isdisjoint(keys.tolist())
        union.update(keys.tolist())
    assert union == seen


def test_keyed_ffm_two_ranks(tmp_path):
    """FFM (39 fields, k=4): rows of Fc * k floats, keyed and sharded"""
    _check_train(tmp_path, "ffm", 6000, 4, 128, 3, 5e-5)


def test_keyed_nfm_two_ranks(tmp_path):
    """NFM: keyed embeddings sharded, dense layers replicated and all-reduced"""
    _check_train(tmp_path, "nfm", 8000, 16, 128, 3, 5e-5)


def test_keyed_fm_two_ranks_seeded(tmp_path):
    """upload_keyed_params with the same arrays on both ranks seeds the sharded table like the single-GPU one"""
    parts, _ = _check_train(tmp_path, "fm", 20000, 16, 256, 3, 2e-5, seeded=True)
    assert sum(len(p["keys"]) for p in parts) >= 20000


def test_keyed_two_ranks_overflow_and_refusals(tmp_path):
    mr.launch("dist_keyed_worker.py", tmp_path, ["--mode", "edge"])
    res = mr.load_json(tmp_path)
    for r, o in enumerate(res):
        assert o["evict_create"] is not None and "key_evict" in o["evict_create"]
        assert o["no_max_nnz_create"] is not None and "max_nnz" in o["no_max_nnz_create"]
        assert o["a_upload"] is None and np.isfinite(o["a_loss"])
        # owner 1's shard overflows: both ranks fail the upload with the same message, naming owner 1
        assert o["b_upload"] is not None and "owner rank 1" in o["b_upload"] and "capacity" in o["b_upload"], o["b_upload"]
        assert isinstance(o["b_step"], str) and "no usable batch" in o["b_step"]
        assert o["kept_rows"]
        assert o["c_upload"] is None and np.isfinite(o["c_loss"])
        assert o["lookup_upload"] is not None and "insert = 0" in o["lookup_upload"]
        assert o["d_upload"] is None and np.isfinite(o["d_loss"])
    assert res[0]["b_upload"] == res[1]["b_upload"]
    assert res[0]["rows_after_b"] == res[0]["rows_after_a"]  # owner 0: no new key in batch B
    assert res[1]["rows_after_b"] == 32                       # owner 1: its shard is full
    assert "insert = 0" in res[0]["mixed_upload"]
    assert "rank 0 refused" in res[1]["mixed_upload"], res[1]["mixed_upload"]
