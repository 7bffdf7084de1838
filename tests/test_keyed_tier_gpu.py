"""Host tier of a keyed context (cfg.key_host_rows, csrc/keys.cu): lctr_evict_keys moves evicted rows with their optimizer
state into pinned host memory, and uploads bring them back bit for bit when their keys return.  A numpy model replays the
upload clock and predicts what eviction does; the model of a tiered context is its device rows plus its tier rows, a key
in at most one of them, and only lctr_evict_host_tier drops one."""
import numpy as np
import pytest

from keyed_model import OPTS, Batch, Clock, bits, history, init_v, model_evict, replay
from keyed_model import rows as _rows
from lightctr_b200.dist import fmix64

pytestmark = pytest.mark.gpu

K_FM, K_NFM, K_FFM, FC_FFM = 8, 16, 3, 5  # FFM rows of 15 floats take the scalar copies


def _ctx(model, cap, opt=0, tier=0, key_evict=True, rows=100):
    from lightctr_b200 import capi
    kw = dict(optimizer=opt, key_mode=capi.KEYS_HASHED, key_evict=key_evict, key_host_rows=tier)
    if model == "fm":
        return capi.Context(capi.MODEL_FM, cap, K_FM, **kw)
    if model == "ffm":
        return capi.Context(capi.MODEL_FFM, cap, K_FFM, FC_FFM, **kw)
    return capi.Context(capi.MODEL_NFM, cap, K_NFM, hidden=(32,), minibatch_size=rows, **kw)


def _by_key(ctx):
    """key -> the six per-row arrays' values of its device row"""
    keys, rows = ctx.download_keys(), _rows(ctx)
    return {k: [a[i] for a in rows] for i, k in enumerate(keys.tolist())}


def _tier(ctx):
    keys, W, V = ctx.download_host_tier()
    return keys, W, V.reshape(len(keys), ctx.rowlen)


def _same_state(ctx, before):
    assert np.array_equal(ctx.download_keys(), before[0])
    for x, y in zip(before[1], _rows(ctx)):
        assert np.array_equal(bits(x), bits(y))
    for x, y in zip(before[2], _tier(ctx)):
        assert np.array_equal(bits(x) if x.dtype != np.uint64 else x, bits(y) if y.dtype != np.uint64 else y)


def _state(ctx):
    return ctx.download_keys(), _rows(ctx), _tier(ctx)


def _same_model(a, b):
    """the same keys in each table with bit-equal rows, whatever the row numbering"""
    ka, kb = _by_key(a), _by_key(b)
    assert sorted(ka) == sorted(kb)
    for k, va in ka.items():
        for x, y in zip(va, kb[k]):
            assert np.array_equal(bits(np.atleast_1d(x)), bits(np.atleast_1d(y)))
    ta, tb = _tier(a), _tier(b)
    ia, ib = np.argsort(ta[0]), np.argsort(tb[0])
    assert np.array_equal(ta[0][ia], tb[0][ib])
    for x, y in zip(ta[1:], tb[1:]):
        assert np.array_equal(bits(x[ia]), bits(y[ib]))


# ---- 1. spill ------------------------------------------------------------------------------------------------------
def test_spill_leaves_the_device_as_an_untiered_eviction_and_keeps_the_rows():
    batches = history(5, 8)
    ctx = _ctx("fm", 4000, OPTS["ftrl"], tier=4000)
    clk = Clock()
    replay(ctx, batches, clk, train=True)
    table = ctx.download_keys()
    n = len(table)
    before = _rows(ctx)
    ev, new = model_evict(table, clk.ages(table), 5, n // 2)
    keys, We, Ve = ctx.evict_keys(5, n // 2, export=True)
    assert 0 < len(keys) < n
    assert np.array_equal(keys, table[ev]) and np.array_equal(ctx.download_keys(), new)
    pos = {k: i for i, k in enumerate(table.tolist())}
    old = np.array([pos[k] for k in new.tolist()])
    for a, b in zip(before, _rows(ctx)):
        assert np.array_equal(bits(b[:len(new)]), bits(a[old]))
    tk, tW, tV = _tier(ctx)
    assert np.array_equal(tk, keys)
    assert np.array_equal(bits(tW), bits(We)) and np.array_equal(bits(tV.ravel()), bits(Ve))
    assert np.array_equal(bits(We), bits(before[0][:n][ev])) and np.array_equal(bits(Ve), bits(before[1][:n][ev].ravel()))
    ctx.close()


# ---- 2. restore ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["fm", "ffm", "nfm"])
@pytest.mark.parametrize("opt", ["adagrad", "ftrl", "ps_adagrad"])
def test_returning_keys_get_their_rows_back_bit_for_bit(model, opt):
    ctx = _ctx(model, 4000, OPTS[opt], tier=4000)
    batches = history(7, 8)
    replay(ctx, batches, train=True)
    before = _by_key(ctx)
    n = len(before)
    gone, _, _ = ctx.evict_keys(max_rows=n // 2, export=True)
    tk0, tW0, tV0 = _tier(ctx)
    assert np.array_equal(tk0, gone)
    rng = np.random.default_rng(1)
    keys = batches[-1].keys.copy()
    back = rng.random(len(keys)) < 0.3
    keys[back] = gone[rng.integers(0, len(gone) // 2, int(back.sum()))]
    Batch(keys, 6, rng).upload(ctx, 0)
    ret = np.intersect1d(np.unique(keys), gone)
    assert len(ret) > 10
    rows, after = ctx.lookup_keys(ret), _rows(ctx)
    assert np.all(rows >= 0)
    for k, r in zip(ret.tolist(), rows.tolist()):
        for a, b in zip(before[k], after):
            assert np.array_equal(bits(np.atleast_1d(a)), bits(np.atleast_1d(b[r])))
    tk, tW, tV = _tier(ctx)
    assert np.array_equal(np.sort(tk), np.setdiff1d(gone, ret))
    p0 = {k: i for i, k in enumerate(tk0.tolist())}
    idx = np.array([p0[k] for k in tk.tolist()])
    assert np.array_equal(bits(tW), bits(tW0[idx])) and np.array_equal(bits(tV), bits(tV0[idx]))
    assert np.isfinite(ctx.train_step(0)[0])
    ctx.close()


# ---- 3. nothing is lost ------------------------------------------------------------------------------------------------
def test_every_uploaded_key_stays_in_exactly_one_table():
    ctx = _ctx("fm", 1200, tier=20000)
    batches = history(3, n_up=16, universe=6000)
    seen = set()
    for i, b in enumerate(batches):
        if i % 3 == 2:
            ctx.evict_keys(max_idle=1)
        ctx.evict_keys(max_rows=1200 - len(np.unique(b.keys)))
        b.upload(ctx, i % 8, insert=(i % 5 != 4))
        if i % 5 != 4:
            seen |= set(b.keys.tolist())
            ctx.train_step(i % 8)
        dev, tier = ctx.download_keys(), ctx.download_host_tier()[0]
        assert len(np.intersect1d(dev, tier)) == 0
        assert set(dev.tolist()) | set(tier.tolist()) == seen
    ctx.close()


# ---- 4. training equivalence -----------------------------------------------------------------------------------------
def _drift(n_batches, unique, seed=9, rows=100, per=5, window=900, shift=150):
    rng = np.random.default_rng(seed)
    pool = fmix64(np.arange(window + shift * n_batches, dtype=np.uint64) + np.uint64(1 << 45))
    out = []
    for i in range(n_batches):
        pick = rng.choice(window, rows * per, replace=False) if unique else rng.integers(0, window, rows * per)
        out.append(Batch(pool[i * shift + pick], per, rng))
    return out


@pytest.mark.parametrize("unique", [True, False])
def test_tiered_training_matches_a_context_that_never_evicts(unique):
    from lightctr_b200 import capi
    cap = 1000
    batches = _drift(14, unique)
    assert len(set(np.concatenate([b.keys for b in batches]).tolist())) > 1.5 * cap
    t = _ctx("fm", cap, tier=10000)
    big = capi.Context(capi.MODEL_FM, 10000, K_FM, key_mode=capi.KEYS_HASHED)
    for i, b in enumerate(batches):
        t.evict_keys(max_rows=cap - len(np.unique(b.keys)))
        b.upload(t, 0)
        b.upload(big, 0)
        lt, lb = t.train_step(0)[0], big.train_step(0)[0]
        assert abs(lt - lb) <= 1e-6 * abs(lb), (i, lt, lb)
        dk = t.download_keys()
        Wt, Vt = t.download_params()
        tk, tW, tV = _tier(t)
        Wb, Vb = big.download_params()
        rd, rt = big.lookup_keys(dk), big.lookup_keys(tk)
        assert np.all(rd >= 0) and np.all(rt >= 0)
        got_W = np.concatenate([Wt[:len(dk)], tW])
        got_V = np.concatenate([Vt.reshape(-1, K_FM)[:len(dk)], tV])
        want_W = Wb[np.concatenate([rd, rt])]
        want_V = Vb.reshape(-1, K_FM)[np.concatenate([rd, rt])]
        if unique:
            assert np.array_equal(bits(got_W), bits(want_W)) and np.array_equal(bits(got_V), bits(want_V)), i
        else:
            assert np.max(np.abs(got_W - want_W)) < 2e-5 and np.max(np.abs(got_V - want_V)) < 2e-5, i
    assert len(t.download_host_tier()[0]) > 0
    t.close(); big.close()


# ---- 5. lookup-only --------------------------------------------------------------------------------------------------
def test_lookup_only_upload_restores_tier_keys_and_keeps_their_stamps():
    from lightctr_b200 import capi
    ctx = _ctx("fm", 4000, tier=4000)
    clk = Clock()
    batches = history(13, 8)
    replay(ctx, batches, clk, train=True)
    gone, _, _ = ctx.evict_keys(max_idle=3, export=True)
    assert len(gone) > 20
    rng = np.random.default_rng(4)
    unseen = fmix64(np.arange(50, dtype=np.uint64) + np.uint64(1 << 50))
    keys = np.concatenate([gone[:40], unseen, batches[-1].keys[:110]])
    rng.shuffle(keys)
    Batch(keys, 5, rng).upload(ctx, 1, insert=False)
    rows = ctx.lookup_keys(gone[:40])
    assert np.all(rows >= 0)
    assert np.all(ctx.lookup_keys(unseen) == -1)
    assert np.array_equal(np.sort(ctx.download_host_tier()[0]), np.sort(gone[40:]))
    with pytest.raises(capi.LctrError, match="insert = 0"):
        ctx.train_step(1)
    assert np.all(np.isfinite(ctx.predict(1)))
    # the clock did not advance and the restored rows kept their tier stamps: the model predicts the next eviction
    table = ctx.download_keys()
    ev, new = model_evict(table, clk.ages(table), 3, None)
    assert np.all(ev[np.isin(table, gone[:40])])
    keys_out, _, _ = ctx.evict_keys(max_idle=3, export=True)
    assert np.array_equal(keys_out, table[ev]) and np.array_equal(ctx.download_keys(), new)
    ctx.close()


# ---- 6. limits -------------------------------------------------------------------------------------------------------
def test_spill_into_a_full_tier_changes_nothing():
    from lightctr_b200 import capi
    rng = np.random.default_rng(17)
    pool = fmix64(np.arange(400, dtype=np.uint64) + np.uint64(77))
    ctx = _ctx("fm", 4000, tier=150)
    replay(ctx, [Batch(pool[100 * i:100 * (i + 1)], 4, rng) for i in range(4)], train=True)  # ages 3, 2, 1, 0
    before = _state(ctx)
    with pytest.raises(capi.LctrError, match=r"150 rows \(cfg.key_host_rows\) with 150 free"):
        ctx.evict_keys(max_idle=0)
    _same_state(ctx, before)
    assert ctx.evict_keys(max_idle=2) == 100
    before = _state(ctx)
    with pytest.raises(capi.LctrError, match="with 50 free"):
        ctx.evict_keys(max_idle=1)
    _same_state(ctx, before)
    assert np.array_equal(np.sort(ctx.download_host_tier()[0]), np.sort(pool[:100]))
    ctx.close()


@pytest.mark.parametrize("insert", [True, False])
def test_restore_past_the_device_capacity_fails_and_keeps_the_keys_in_the_tier(insert):
    from lightctr_b200 import capi
    cap = 700
    ctx = _ctx("fm", cap, tier=4000)
    rng = np.random.default_rng(6)
    pool = fmix64(np.arange(3000, dtype=np.uint64) + np.uint64(1 << 40))
    Batch(pool[:600], 6, rng).upload(ctx, 0)
    gone, _, _ = ctx.evict_keys(max_rows=0, export=True)
    assert len(gone) == 600
    Batch(pool[1000:1600], 6, rng).upload(ctx, 0)  # 100 rows left
    k0, W0, V0 = _tier(ctx)
    at = {k: i for i, k in enumerate(k0.tolist())}
    back = Batch(pool[:300], 6, rng)
    with pytest.raises(capi.LctrError, match="capacity of %d rows" % cap):
        back.upload(ctx, 1, insert=insert)
    dev, tier = ctx.download_keys(), ctx.download_host_tier()[0]
    assert len(dev) == cap and len(tier) == 500
    assert len(np.intersect1d(dev, tier)) == 0
    assert set(dev.tolist()) | set(tier.tolist()) == set(pool[:600].tolist()) | set(pool[1000:1600].tolist())

    def tier_unchanged():  # every key left in the tier keeps its row bit for bit
        k, W, V = _tier(ctx)
        idx = np.array([at[x] for x in k.tolist()])
        assert np.array_equal(bits(W), bits(W0[idx])) and np.array_equal(bits(V), bits(V0[idx]))
        return k

    tier_unchanged()
    # the same upload again: the keys refused before are still refused, none slips to the null row
    with pytest.raises(capi.LctrError, match="capacity of %d rows" % cap):
        back.upload(ctx, 1, insert=insert)
    assert np.array_equal(np.sort(tier_unchanged()), np.sort(tier))
    assert np.array_equal(np.sort(ctx.download_keys()), np.sort(dev))
    ctx.close()


def test_spills_past_half_the_index_rebuild_it_and_lose_nothing():
    # a tier of 100 rows has an index of 256 slots, rebuilt by a spill once live plus dead slots pass 128
    ctx = _ctx("fm", 1000, tier=100)
    rng = np.random.default_rng(8)
    pool = fmix64(np.arange(200, dtype=np.uint64) + np.uint64(1 << 41))
    A, B = Batch(pool[:100], 4, rng), Batch(pool[100:], 4, rng)
    A.upload(ctx, 0)
    ctx.train_step(0)
    B.upload(ctx, 1)
    ctx.train_step(1)
    before = _by_key(ctx)

    def same_rows(keys):
        rows, after = ctx.lookup_keys(keys), _rows(ctx)
        assert np.all(rows >= 0)
        for key, r in zip(keys.tolist(), rows.tolist()):
            for x, y in zip(before[key], after):
                assert np.array_equal(bits(np.atleast_1d(x)), bits(np.atleast_1d(y[r])))

    assert ctx.evict_keys(max_idle=0) == 100  # A: 100 slots claimed
    assert np.array_equal(np.sort(ctx.download_host_tier()[0]), np.sort(A.keys))
    A.upload(ctx, 0)  # A back: 100 dead slots
    same_rows(A.keys)
    assert len(ctx.download_host_tier()[0]) == 0
    assert ctx.evict_keys(max_idle=0) == 100  # B: 100 more slots, 200 > 128, so this spill rebuilds the index
    tk, tW, tV = _tier(ctx)
    assert np.array_equal(np.sort(tk), np.sort(B.keys))
    B.upload(ctx, 1, insert=False)  # found through the rebuilt index
    same_rows(B.keys)
    assert len(ctx.download_host_tier()[0]) == 0
    assert set(ctx.download_keys().tolist()) == set(pool.tolist())
    ctx.close()


def test_evict_host_tier_follows_the_rule_on_tier_stamps():
    ctx = _ctx("fm", 4000, tier=4000)
    clk = Clock()
    batches = history(19, n_up=10)
    for i, b in enumerate(batches):
        b.upload(ctx, 0)
        clk.insert(b.keys)
        if i % 3 == 2:
            ctx.evict_keys(max_idle=1)
    tier, tW, tV = _tier(ctx)
    ages = clk.ages(tier)
    assert len(np.unique(ages)) > 2
    ev, new = model_evict(tier, ages, 7, int(len(tier) * 0.4))
    assert 0 < ev.sum() < len(tier)
    keys, W, V = ctx.evict_host_tier(7, int(len(tier) * 0.4), export=True)
    assert np.array_equal(keys, tier[ev])
    assert np.array_equal(bits(W), bits(tW[ev])) and np.array_equal(bits(V), bits(tV[ev].ravel()))
    tk, tW2, _ = _tier(ctx)
    assert np.array_equal(tk, new)
    pos = {k: i for i, k in enumerate(tier.tolist())}
    assert np.array_equal(bits(tW2), bits(tW[[pos[k] for k in new.tolist()]]))
    # the freed keys left the model: they come back as new keys, the kept ones from the tier
    back = np.concatenate([keys[:5], new[:5]])
    Batch(back, 2, np.random.default_rng(0)).upload(ctx, 1)
    W_dev, V_dev = ctx.download_params()
    r = ctx.lookup_keys(back)
    assert np.all(W_dev[r[:5]] == 0)
    assert np.max(np.abs(V_dev.reshape(-1, K_FM)[r[:5]] - init_v(keys[:5], K_FM, 0, 1 / np.sqrt(K_FM)))) < 1e-6
    assert np.array_equal(bits(W_dev[r[5:]]), bits(tW2[:5]))
    ctx.close()


# ---- 7. checkpoint -------------------------------------------------------------------------------------------------
def test_checkpoint_round_trip_and_refusals(tmp_path):
    from lightctr_b200 import capi
    batches = history(23, 8)
    a = _ctx("fm", 4000, OPTS["ftrl"], tier=3000)
    replay(a, batches, train=True)
    a.evict_keys(max_idle=2)
    path = str(tmp_path / "tiered.ckpt")
    a.save_checkpoint(path)
    b = _ctx("fm", 4000, OPTS["ftrl"], tier=3000)
    b.load_checkpoint(path)
    _same_state(b, _state(a))
    rng = np.random.default_rng(2)
    once = Batch(rng.permutation(np.unique(batches[0].keys))[:480], 6, rng)  # no repeats: one gradient term per row
    assert len(np.intersect1d(once.keys, a.download_host_tier()[0])) > 10
    for c in (a, b):  # returning keys bring back the same optimizer state
        once.upload(c, 0)
        c.train_step(0)
    _same_model(a, b)
    # refused loads, each leaving the context as it was
    u = _ctx("fm", 4000, OPTS["ftrl"])
    replay(u, batches[:3], train=True)
    upath = str(tmp_path / "untiered.ckpt")
    u.save_checkpoint(upath)
    small = _ctx("fm", 4000, OPTS["ftrl"], tier=10)
    replay(small, batches[:2], train=True)
    for ctx, p, msg in [(u, path, "different trainer"), (b, upath, "different trainer"), (small, path, "key_host_rows = 10")]:
        before = _state(ctx) if ctx is not u else (ctx.download_keys(), _rows(ctx))
        with pytest.raises(capi.LctrError, match=msg):
            ctx.load_checkpoint(p)
        if ctx is u:
            assert np.array_equal(ctx.download_keys(), before[0])
            for x, y in zip(before[1], _rows(ctx)):
                assert np.array_equal(bits(x), bits(y))
        else:
            _same_state(ctx, before)
    a.close(); b.close(); u.close(); small.close()


# ---- 8. rejections and bytes -----------------------------------------------------------------------------------------
def test_rejections_and_device_bytes():
    from lightctr_b200 import capi
    with pytest.raises(capi.LctrError, match="key_host_rows"):
        capi.Context(capi.MODEL_FM, 1000, 8, key_host_rows=100)
    with pytest.raises(capi.LctrError, match="key_host_rows"):
        _ctx("fm", 1000, tier=100, key_evict=False)
    with pytest.raises(capi.LctrError, match="key_host_rows"):
        capi.Context(capi.MODEL_FM, 1000, 8, key_mode=capi.KEYS_HASHED, key_evict=True, key_host_rows=100, world=2,
                     max_nnz=1000)
    untiered = _ctx("fm", 1000)
    with pytest.raises(capi.LctrError, match="host tier"):
        untiered.evict_host_tier(max_idle=0)
    with pytest.raises(capi.LctrError, match="host tier"):
        untiered.download_host_tier()
    cap, rows = 100000, 30000
    t = _ctx("fm", cap, tier=rows)
    u = _ctx("fm", cap)
    T = 16
    while T < 2 * rows:
        T *= 2
    assert t.device_bytes()[0] - u.device_bytes()[0] == T * 12
    Tk = 16
    while Tk < 2 * cap:
        Tk *= 2
    assert u.device_bytes()[0] == (cap + 1) * (K_FM + 1) * 4 * 2 + Tk * 12 + cap * 8 + cap * 8
    t.close(); u.close(); untiered.close()
