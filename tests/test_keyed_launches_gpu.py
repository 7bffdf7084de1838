"""Kernel launches of every keyed call (csrc/keys.cu), counted by lctr_launch_count on small FM and FFM contexts.  The
FM rows of 8 floats take the 16-byte row copies, the FFM rows of 15 the scalar ones.  The counts pin the launch
sequence of each call: a change to how keys.cu issues its kernels must leave them as they are."""
import numpy as np
import pytest

from lightctr_b200.dist import fmix64

pytestmark = pytest.mark.gpu

K_FM, K_FFM, FC_FFM = 8, 3, 5

# launches per call; an upload's count includes the slot preparation after the translation (more of it for FM)
EXPECTED = {
    "fm": {
        "insert_new": 9, "insert_known": 9, "lookup_only": 7, "upload_keyed_params": 5, "evict": 7, "evict_export": 10,
        "load_checkpoint": 1, "evict_tiered": 8, "insert_restore": 11, "lookup_restore": 12, "evict_host_tier": 8,
        "admit_dropped": 9, "admit_kept": 10, "decay": 1,
    },
    "ffm": {
        "insert_new": 4, "insert_known": 4, "lookup_only": 2, "upload_keyed_params": 5, "evict": 7, "evict_export": 10,
        "load_checkpoint": 1, "evict_tiered": 8, "insert_restore": 6, "lookup_restore": 7, "evict_host_tier": 8,
        "admit_dropped": 9, "admit_kept": 5, "decay": 1,
    },
}


def _ctx(model, tier=0):
    from lightctr_b200 import capi
    kw = dict(key_mode=capi.KEYS_HASHED, key_evict=True, key_host_rows=tier)
    if model == "fm":
        return capi.Context(capi.MODEL_FM, 2000, K_FM, **kw)
    return capi.Context(capi.MODEL_FFM, 2000, K_FFM, FC_FFM, **kw)


def _upload(ctx, keys, slot=0, insert=True):
    keys = np.ascontiguousarray(keys, np.uint64)
    rp = np.arange(0, len(keys) + 1, 4, dtype=np.int64)
    fld = (np.arange(len(keys)) % FC_FFM).astype(np.uint16) if ctx.Fc else None
    lab = (np.arange(len(rp) - 1) % 3 == 0).astype(np.int32)
    ctx.upload_batch_keys(slot, rp, keys, fld, None, lab, insert=insert)


def _deltas(model, tmp_path):
    out = {}

    def count(name, ctx, fn):
        before = ctx.launch_count()
        fn()
        out[name] = ctx.launch_count() - before

    pool = fmix64(np.arange(1200, dtype=np.uint64) + np.uint64(1 << 36))
    A, B, C = pool[:400], pool[400:800], pool[800:]
    rowlen = K_FM if model == "fm" else K_FFM * FC_FFM

    ctx = _ctx(model)
    count("insert_new", ctx, lambda: _upload(ctx, A))
    count("insert_known", ctx, lambda: _upload(ctx, A))
    count("lookup_only", ctx, lambda: _upload(ctx, np.concatenate([A[:200], C[:200]]), slot=1, insert=False))
    keys = np.concatenate([A[:50], C[:50]])
    count("upload_keyed_params", ctx, lambda: ctx.upload_keyed_params(keys, np.ones(100), np.ones(100 * rowlen)))
    _upload(ctx, B)
    count("evict", ctx, lambda: ctx.evict_keys(max_idle=0))
    _upload(ctx, A)
    _upload(ctx, C)
    count("evict_export", ctx, lambda: ctx.evict_keys(max_idle=1, max_rows=500, export=True))
    assert np.array_equal(np.sort(ctx.download_keys()), np.sort(C))
    path = str(tmp_path / ("%s.ckpt" % model))
    ctx.save_checkpoint(path)
    count("load_checkpoint", ctx, lambda: ctx.load_checkpoint(path))
    ctx.close()

    ctx = _ctx(model, tier=2000)
    _upload(ctx, A)
    _upload(ctx, B)
    count("evict_tiered", ctx, lambda: ctx.evict_keys(max_idle=0))
    count("insert_restore", ctx, lambda: _upload(ctx, np.concatenate([A[:100], C[:100]])))
    count("lookup_restore", ctx, lambda: _upload(ctx, np.concatenate([A[100:200], C[200:300]]), slot=1, insert=False))
    _upload(ctx, C)
    ctx.evict_keys(max_idle=0)
    count("evict_host_tier", ctx, lambda: ctx.evict_host_tier(max_rows=100))
    ctx.close()

    ctx = _ctx(model)
    ctx.set_key_admission(2, 12)
    count("admit_dropped", ctx, lambda: _upload(ctx, A))
    assert ctx.key_admission_stats() == (len(A), 0)
    count("admit_kept", ctx, lambda: _upload(ctx, A))
    assert ctx.key_admission_stats() == (0, len(A))
    count("decay", ctx, lambda: ctx.decay_key_admission(1))
    ctx.close()
    return out


@pytest.mark.parametrize("model", ["fm", "ffm"])
def test_keyed_calls_issue_the_same_launches(model, tmp_path):
    assert _deltas(model, tmp_path) == EXPECTED[model]
