"""Frequency admission of keyed contexts (lctr_set_key_admission, csrc/keys.cu): a new key gets a row only once
insert-uploads have met it min_count times, counted in a 4-row count-min sketch; entries of keys not admitted leave the
batch, rows stay.  A numpy restatement of the sketch (the cell formula of include/lightctr_b200.h) and of the admission
rule predicts the admitted set, the drop counts, and the batch the step kernels must see."""
import math

import numpy as np
import pytest

from keyed_model import cells
from lightctr_b200.dist import fmix64

pytestmark = pytest.mark.gpu

FC = 39  # fields of the FFM cases, as the C2 stream has
CAP = 50000


class Admit:
    """numpy model of one context's admission: the sketch, the present keys (device rows) and the tier's keys"""

    def __init__(self, min_count, lw):
        self.m, self.lw = min_count, lw
        self.sk = np.zeros((4, 1 << lw), np.uint64)
        self.present, self.tier = set(), set()

    def upload(self, keys):
        """one insert-upload: the keep mask over the entries, dropped entries, admitted keys"""
        keys = np.asarray(keys, np.uint64)
        known = self.present | self.tier
        absent = np.array([k not in known for k in keys.tolist()], bool)
        cs = cells(keys[absent], self.lw)
        for i in range(4):
            np.add.at(self.sk[i], cs[i], 1)
        new = np.unique(keys[absent])
        cn = cells(new, self.lw)
        cnt = np.min(np.stack([self.sk[i][cn[i]] for i in range(4)]), axis=0) if len(new) else np.zeros(0, np.uint64)
        admitted = set(new[cnt >= self.m].tolist())
        restored = set(keys.tolist()) & self.tier
        self.tier -= restored
        self.present |= admitted | restored
        keep = np.array([k in self.present for k in keys.tolist()], bool)
        return keep, int((~keep).sum()), len(admitted)

    def decay(self, shift):
        self.sk = np.zeros_like(self.sk) if shift >= 32 else self.sk >> np.uint64(shift)


class Batch:
    """rows of ragged length over the first fields, key of field f from a Zipf(1.1) draw inside that field; the last
    `lonely` rows hold keys met nowhere else, so they lose every entry while admission is on"""

    def __init__(self, rng, rows, fields, lonely=0, with_val=False, distinct=False, base=0):
        lens = rng.integers(1, fields + 1, rows)
        rp = np.zeros(rows + 1, np.int64)
        rp[1:] = np.cumsum(lens)
        fld = np.concatenate([np.arange(n) for n in lens]).astype(np.uint16)
        if distinct:  # every key once in the batch: each gradient row gets one contribution, so training is bit-exact
            z = np.arange(rp[-1], dtype=np.uint64) + np.uint64(base)
        else:
            z = np.minimum(rng.zipf(1.1, rp[-1]), 1 << 20).astype(np.uint64)
        keys = fmix64((fld.astype(np.uint64) << np.uint64(32)) + z)
        for r in range(rows - lonely, rows):
            keys[rp[r]:rp[r + 1]] = fmix64(np.uint64(1 << 60) + np.uint64(base) + np.arange(rp[r], rp[r + 1], dtype=np.uint64))
        self.rp, self.keys, self.fld = rp, keys, fld
        self.val = (rng.random(len(keys)) * 2).astype(np.float32) if with_val else None
        self.lab = (rng.random(rows) < 0.3).astype(np.int32)

    def upload(self, ctx, slot, insert=True):
        ctx.upload_batch_keys(slot, self.rp, self.keys, self.fld if ctx.Fc else None, self.val, self.lab, insert=insert)

    def filtered(self, keep):
        """the batch with the entries of `keep` only, in order, every row kept"""
        b = Batch.__new__(Batch)
        per = np.add.reduceat(keep.astype(np.int64), self.rp[:-1]) if len(keep) else np.zeros(len(self.rp) - 1, np.int64)
        per[np.diff(self.rp) == 0] = 0
        b.rp = np.concatenate([[0], np.cumsum(per)]).astype(np.int64)
        b.keys, b.fld = self.keys[keep], self.fld[keep]
        b.val = None if self.val is None else self.val[keep]
        b.lab = self.lab
        return b


def _ctx(model, cap=CAP, **kw):
    from lightctr_b200 import capi
    kw = dict(key_mode=capi.KEYS_HASHED, **kw)
    if model == "fm":
        return capi.Context(capi.MODEL_FM, cap, 16, **kw)
    if model == "ffm":
        return capi.Context(capi.MODEL_FFM, cap, 4, FC, **kw)
    return capi.Context(capi.MODEL_NFM, cap, 16, hidden=(32,), minibatch_size=256, **kw)


def _fields(model):
    return FC if model == "ffm" else 8


def _by_key(ctx):
    keys = ctx.download_keys()
    W, V = ctx.download_params()
    r = ctx.rowlen
    return {k: (W[i], V[i * r:(i + 1) * r]) for i, k in enumerate(keys.tolist())}


@pytest.mark.parametrize("model", ["fm", "ffm", "nfm"])
def test_admitted_set_follows_the_model(model):
    """Over a Zipf history the rows held are exactly the model's present set after every upload, and the stats are the
    model's drop and admit counts; a narrow sketch (2^10) makes the model reproduce collisions too."""
    rng = np.random.default_rng(1)
    ctx = _ctx(model)
    ctx.set_key_admission(3, 10)
    m = Admit(3, 10)
    seen, total_dropped = set(), 0
    for i in range(6):
        b = Batch(rng, 256, _fields(model), lonely=4)
        b.upload(ctx, i % 8)
        _, dropped, admitted = m.upload(b.keys)
        seen |= set(b.keys.tolist())
        total_dropped += dropped
        assert set(ctx.download_keys().tolist()) == m.present, i
        assert ctx.key_admission_stats() == (dropped, admitted), i
        loss, _ = ctx.train_step(i % 8)
        assert math.isfinite(loss)
    assert total_dropped > 0 and 0 < len(m.present) < len(seen)
    ctx.close()


@pytest.mark.parametrize("model,with_val", [("fm", False), ("fm", True), ("ffm", False), ("ffm", True), ("nfm", True)])
def test_compaction_equals_the_host_filtered_batch(model, with_val):
    """A context with admission uploading the raw batch and one without uploading the batch the model keeps, both seeded
    with the same keys, predict the same pCTR bit for bit and train to the same parameters per key."""
    rng = np.random.default_rng(2)
    b = Batch(rng, 256, _fields(model), lonely=6, with_val=with_val)
    uniq, cnt = np.unique(b.keys, return_counts=True)
    seed = uniq[np.argsort(-cnt)[:40]]  # the most frequent keys already have rows on both sides
    a, o = _ctx(model), _ctx(model)
    a.set_key_admission(2, 14)
    for c in (a, o):
        c.upload_keyed_params(seed)
    m = Admit(2, 14)
    m.present |= set(seed.tolist())
    keep, dropped, admitted = m.upload(b.keys)
    f = b.filtered(keep)
    assert dropped > 0 and np.sum(np.diff(f.rp) == 0) >= 6  # rows that lose every entry
    b.upload(a, 0)
    f.upload(o, 0)
    assert a.key_admission_stats() == (dropped, admitted)
    assert set(a.download_keys().tolist()) == set(o.download_keys().tolist()) == m.present
    if model != "nfm":  # (no NFM predictor)
        pa, po = a.predict(0), o.predict(0)
        assert np.array_equal(pa.view(np.uint32), po.view(np.uint32))
        assert np.array_equal(a.download_pred(0).view(np.uint32), po.view(np.uint32))
    for _ in range(3):
        la, ca = a.train_step(0)
        lo, co = o.train_step(0)
        assert abs(la - lo) <= 1e-5 * abs(lo) and ca == co, (la, lo)
    ga, go = _by_key(a), _by_key(o)
    assert set(ga) == set(go)
    dw = max(abs(float(ga[k][0]) - float(go[k][0])) for k in go)
    dv = max(float(np.max(np.abs(ga[k][1] - go[k][1]))) for k in go)
    assert dw < 5e-5 and dv < 5e-5, (dw, dv)
    a.close()
    o.close()


def test_all_entries_dropped_trains_rows_without_entries():
    """A batch whose every key is new and seen once keeps its rows and loses every entry: FM loss rows * ln 2."""
    rng = np.random.default_rng(3)
    ctx = _ctx("fm")
    ctx.set_key_admission(2, 12)
    b = Batch(rng, 64, 8, lonely=64)
    b.upload(ctx, 0)
    assert ctx.key_admission_stats() == (len(b.keys), 0)
    assert len(ctx.download_keys()) == 0
    loss, correct = ctx.train_step(0)
    assert abs(loss - 64 * math.log(2.0)) <= 1e-5 * 64 * math.log(2.0) and correct == 0
    p = ctx.predict(0)
    assert len(p) == 64 and np.all(p == np.float32(0.5))
    ctx.close()


def _one(keys):
    """one row holding the given keys"""
    keys = np.asarray(keys, np.uint64)
    return np.array([0, len(keys)], np.int64), keys, np.array([1], np.int32)


def _up(ctx, keys, insert=True, slot=0):
    rp, k, lab = _one(keys)
    ctx.upload_batch_keys(slot, rp, k, None, None, lab, insert=insert)


def test_tier_keys_are_restored_whatever_their_count():
    ctx = _ctx("fm", cap=1000, key_evict=True, key_host_rows=1000)
    ctx.set_key_admission(2, 10)
    A = fmix64(np.arange(10, dtype=np.uint64) + np.uint64(7))
    _up(ctx, np.concatenate([A, A]))  # entries, not distinct keys, are counted: admitted at once
    assert ctx.key_admission_stats() == (0, 10) and set(ctx.download_keys().tolist()) == set(A.tolist())
    assert ctx.evict_keys(max_rows=0) == 10
    ctx.set_key_admission(2, 10)  # a zero sketch: only the tier can bring them back
    fresh = fmix64(np.uint64(99999))
    _up(ctx, np.concatenate([A, [fresh]]))
    assert ctx.key_admission_stats() == (1, 0)
    assert set(ctx.download_keys().tolist()) == set(A.tolist())
    assert len(ctx.download_host_tier()[0]) == 0
    ctx.close()


def test_upload_keyed_params_bypasses_admission():
    ctx = _ctx("fm")
    ctx.set_key_admission(5, 10)
    A = fmix64(np.arange(20, dtype=np.uint64) + np.uint64(3))
    ctx.upload_keyed_params(A)
    assert set(ctx.download_keys().tolist()) == set(A.tolist())
    _up(ctx, A)
    assert ctx.key_admission_stats() == (0, 0)
    ctx.close()


def test_lookup_uploads_count_nothing():
    ctx = _ctx("fm")
    ctx.set_key_admission(2, 10)
    x = fmix64(np.array([42], np.uint64))
    for _ in range(3):
        _up(ctx, x, insert=False)
    _up(ctx, x)
    assert ctx.key_admission_stats() == (1, 0) and len(ctx.download_keys()) == 0
    _up(ctx, x)
    assert ctx.key_admission_stats() == (0, 1) and ctx.download_keys().tolist() == x.tolist()
    ctx.close()


def test_dropped_keys_stamp_nothing():
    ctx = _ctx("fm", key_evict=True)
    ctx.set_key_admission(2, 10)
    a, b = fmix64(np.array([1, 2], np.uint64))
    _up(ctx, [a, a, b])   # clock 1: a admitted and stamped; b counted once, dropped
    _up(ctx, [b, a])      # clock 2: b admitted; both rows kept entries and are stamped
    assert ctx.key_admission_stats() == (0, 1)
    c = fmix64(np.array([3], np.uint64))
    _up(ctx, [c])         # clock 3: c dropped, nothing stamped
    assert ctx.key_admission_stats() == (1, 0)
    assert ctx.evict_keys(max_idle=0) == 2  # both rows are one upload old: the dropped key stamped nothing
    ctx.close()


def test_evicted_key_returns_at_once_then_must_earn_it_after_decay():
    ctx = _ctx("fm", key_evict=True)
    ctx.set_key_admission(2, 10)
    x = fmix64(np.array([5], np.uint64))
    _up(ctx, [x[0], x[0]])
    assert ctx.download_keys().tolist() == x.tolist()
    assert ctx.evict_keys(max_rows=0) == 1
    _up(ctx, x)  # its counters are still 2
    assert ctx.key_admission_stats() == (0, 1) and ctx.download_keys().tolist() == x.tolist()
    assert ctx.evict_keys(max_rows=0) == 1
    ctx.decay_key_admission(32)
    _up(ctx, x)
    assert ctx.key_admission_stats() == (1, 0) and len(ctx.download_keys()) == 0
    _up(ctx, x)
    assert ctx.key_admission_stats() == (0, 1)
    ctx.close()


def test_decay_matches_the_model():
    rng = np.random.default_rng(4)
    ctx = _ctx("fm")
    ctx.set_key_admission(4, 10)
    m = Admit(4, 10)
    for i in range(6):
        if i in (2, 4):
            ctx.decay_key_admission(1 if i == 2 else 3)
            m.decay(1 if i == 2 else 3)
        b = Batch(rng, 128, 8)
        b.upload(ctx, 0)
        _, dropped, admitted = m.upload(b.keys)
        assert ctx.key_admission_stats() == (dropped, admitted), i
        assert set(ctx.download_keys().tolist()) == m.present, i
    ctx.close()


def test_admitted_keys_past_the_capacity_fail_as_new_keys_do():
    from lightctr_b200 import capi
    ctx = _ctx("fm", cap=8)  # 16 table slots: 12 keys find slots, 4 of them no row
    ctx.set_key_admission(2, 10)
    A = fmix64(np.arange(12, dtype=np.uint64) + np.uint64(11))
    _up(ctx, A)  # counted once: nothing admitted, nothing fails
    assert len(ctx.download_keys()) == 0
    with pytest.raises(capi.LctrError, match="capacity of 8 rows"):
        _up(ctx, A)
    ctx.close()


def _run_history(ctx, batches):
    counts = []
    for i, b in enumerate(batches):
        n0 = ctx.launch_count()
        b.upload(ctx, i % 8)
        ctx.train_step(i % 8)
        counts.append(ctx.launch_count() - n0)
    return counts


@pytest.mark.parametrize("model", ["fm", "ffm"])
def test_off_means_off(model):
    """min_count = 1, and admission switched off again, launch and train exactly as a context that never set it (every
    key once per batch, so each gradient row gets one contribution and the parameters compare bit for bit)."""
    rng = np.random.default_rng(5)
    batches = [Batch(rng, 64, _fields(model), distinct=True, base=1000 * (i % 3)) for i in range(5)]
    ctxs = [_ctx(model) for _ in range(3)]
    ctxs[1].set_key_admission(1, 12)
    ctxs[2].set_key_admission(3, 12)
    ctxs[2].set_key_admission(0, 0)
    runs = [_run_history(c, batches) for c in ctxs]
    assert runs[0] == runs[1] == runs[2]

    def by_key(c):  # rows follow arrival order: W, V, s1, s2 of every row, sorted by key
        keys = c.download_keys()
        o, n, r = np.argsort(keys), len(keys), c.rowlen
        F = c.F
        W, V = c.download_params()
        s1, s2 = c.download_opt_state()
        parts = [W[:n], V.reshape(F, r)[:n], s1[:n], s1[F:].reshape(F, r)[:n], s2[:n], s2[F:].reshape(F, r)[:n]]
        return keys[o], [p[o] for p in parts]

    ref = by_key(ctxs[0])
    for c in ctxs[1:]:
        got = by_key(c)
        assert np.array_equal(got[0], ref[0])
        for x, y in zip(got[1], ref[1]):
            assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    assert ctxs[1].device_bytes() == ctxs[0].device_bytes()
    for c in ctxs:
        c.close()


def test_sketch_counts_in_device_bytes():
    ctx = _ctx("fm")
    base = ctx.device_bytes()[0]
    ctx.set_key_admission(2, 16)
    assert ctx.device_bytes()[0] == base + 16 * (1 << 16)
    ctx.set_key_admission(1, 16)
    assert ctx.device_bytes()[0] == base
    ctx.close()


def _header_word(path):
    with open(path, "rb") as f:
        return int(np.frombuffer(f.read(24)[20:24], np.int32)[0])


def test_checkpoint_round_trip_admits_what_the_original_admits(tmp_path):
    from lightctr_b200 import capi
    rng = np.random.default_rng(6)
    batches = [Batch(rng, 128, 8, lonely=2) for _ in range(6)]
    a = _ctx("fm")
    a.set_key_admission(3, 11)
    for i, b in enumerate(batches[:3]):
        b.upload(a, 0)
        a.train_step(0)
    path = str(tmp_path / "a.ckpt")
    a.save_checkpoint(path)
    assert _header_word(path) & 0x400
    saved_keys = a.download_keys()
    r = _ctx("fm")
    r.set_key_admission(3, 11)
    r.load_checkpoint(path)
    assert np.array_equal(r.download_keys(), saved_keys)
    for b in batches[3:]:
        b.upload(a, 0)
        b.upload(r, 0)
        assert r.key_admission_stats() == a.key_admission_stats()
        assert set(r.download_keys().tolist()) == set(a.download_keys().tolist())  # rows follow arrival order

    # other settings, or none, are refused before anything changes
    for mc, lw, theirs in ((2, 11, "min_count 2, log2_width 11"), (3, 12, "min_count 3, log2_width 12"), (1, 0, "off")):
        x = _ctx("fm")
        x.set_key_admission(mc, lw)
        batches[0].upload(x, 0)
        before = x.download_keys(), x.download_params()
        with pytest.raises(capi.LctrError, match="min_count 3, log2_width 11.*" + theirs):
            x.load_checkpoint(path)
        assert np.array_equal(x.download_keys(), before[0])
        for p, q in zip(x.download_params(), before[1]):
            assert np.array_equal(p.view(np.uint32), q.view(np.uint32))
        x.close()

    # resharding into a context without admission skips the sketch
    s = _ctx("fm")
    s.load_checkpoint_shards([path])
    assert np.array_equal(s.download_keys(), saved_keys)
    assert s.key_admission_stats() == (0, 0)
    # ... and one with other settings refuses
    t = _ctx("fm")
    t.set_key_admission(2, 11)
    with pytest.raises(capi.LctrError, match="key admission"):
        t.load_checkpoint_shards([path])
    for c in (a, r, s, t):
        c.close()


def test_files_without_admission_keep_their_bytes(tmp_path):
    rng = np.random.default_rng(8)
    b = Batch(rng, 64, 8)
    c = _ctx("fm")
    b.upload(c, 0)
    p1, p2 = str(tmp_path / "1.ckpt"), str(tmp_path / "2.ckpt")
    c.save_checkpoint(p1)
    c.set_key_admission(2, 10)
    c.set_key_admission(1, 10)
    c.save_checkpoint(p2)
    assert open(p1, "rb").read() == open(p2, "rb").read()
    assert not _header_word(p1) & 0x400
    c.close()


def test_refusals():
    from lightctr_b200 import capi
    dense = capi.Context(capi.MODEL_FM, 1000, 16)
    with pytest.raises(capi.LctrError, match="key_mode"):
        dense.set_key_admission(2, 12)
    dense.close()
    two = capi.Context(capi.MODEL_FM, 1000, 16, world=2, rank=0, minibatch_size=64, max_nnz=1024, key_mode=capi.KEYS_HASHED)
    with pytest.raises(capi.LctrError, match="world = 2"):
        two.set_key_admission(2, 12)
    two.close()
    wnd = capi.Context(capi.MODEL_WND, 1000, 4, 3, hidden=(8,), key_mode=capi.KEYS_HASHED)
    with pytest.raises(capi.LctrError, match="Wide&Deep"):
        wnd.set_key_admission(2, 12)
    wnd.close()
    ctx = _ctx("fm")
    for lw in (9, 29):
        with pytest.raises(capi.LctrError, match="log2_width = %d outside" % lw):
            ctx.set_key_admission(2, lw)
    with pytest.raises(capi.LctrError, match="admission is off"):
        ctx.decay_key_admission(1)
    ctx.set_key_admission(2, 10)
    with pytest.raises(capi.LctrError, match="shift = 0 outside"):
        ctx.decay_key_admission(0)
    ctx.close()
