"""Eviction of idle keyed rows (cfg.key_evict = 1, lctr_evict_keys in csrc/keys.cu).  A numpy model replays the upload
history (the clock counts insert-uploads; every row an upload meets is stamped with it) and predicts the evicted set,
the export order and the renumbered table from the table as it stood before the call.  Survivors must keep parameters and
optimizer state bit for bit, training must go on as on a fresh context seeded with the survivors, and the capacity, slot
staleness, checkpoints and refused calls behave as include/lightctr_b200.h states."""
import ctypes as C
import os

import numpy as np
import pytest

from keyed_model import OPTS, Batch, Clock, bits, history, init_v, model_evict, replay
from keyed_model import rows as _rows
from lightctr_b200.dist import fmix64

pytestmark = pytest.mark.gpu

K_FM, K_NFM, K_FFM, FC_FFM = 8, 16, 3, 5  # FFM rows of 15 floats take the scalar path of the row move


def _ctx(model, cap, opt=0, key_evict=True, rows=100):
    from lightctr_b200 import capi
    if model == "fm":
        return capi.Context(capi.MODEL_FM, cap, K_FM, optimizer=opt, key_mode=capi.KEYS_HASHED, key_evict=key_evict)
    if model == "ffm":
        return capi.Context(capi.MODEL_FFM, cap, K_FFM, FC_FFM, optimizer=opt, key_mode=capi.KEYS_HASHED, key_evict=key_evict)
    return capi.Context(capi.MODEL_NFM, cap, K_NFM, optimizer=opt, hidden=(32,), minibatch_size=rows,
                        key_mode=capi.KEYS_HASHED, key_evict=key_evict)


# ---- 1. policy -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model", ["fm", "ffm", "nfm"])
@pytest.mark.parametrize("rule", ["idle", "rows", "both"])
def test_policy_matches_the_model_of_the_upload_history(model, rule):
    batches = history(11, 12)
    ctx = _ctx(model, 4000)
    clk = Clock()
    replay(ctx, batches, clk)
    table = ctx.download_keys()
    ages = clk.ages(table)
    n = len(table)
    max_idle, max_rows = {"idle": (4, None), "rows": (None, int(n * 0.6)), "both": (6, int(n * 0.45))}[rule]
    if rule == "both":  # both limits bind
        assert (ages > max_idle).any() and (ages <= max_idle).sum() > max_rows
    ev, new = model_evict(table, ages, max_idle, max_rows)
    assert 0 < ev.sum() < n
    keys, W, V = ctx.evict_keys(max_idle, max_rows, export=True)
    assert np.array_equal(keys, table[ev])  # ascending order of the old row
    assert len(W) == ev.sum() and len(V) == ev.sum() * ctx.rowlen
    assert np.array_equal(ctx.download_keys(), new)
    assert np.all(ctx.lookup_keys(table[ev]) == -1)
    assert np.array_equal(ctx.lookup_keys(new), np.arange(len(new)))
    ctx.close()


def test_ties_at_the_cutoff_leave_together():
    rng = np.random.default_rng(2)
    pool = fmix64(np.arange(300, dtype=np.uint64) + np.uint64(99))
    batches = [Batch(pool[100 * i:100 * (i + 1)], 4, rng) for i in range(3)]  # ages 2, 1, 0 for 100 rows each
    ctx = _ctx("fm", 1000)
    replay(ctx, batches)
    # max_rows = 150 falls inside the age-1 group: the whole group leaves with the age-2 group
    assert ctx.evict_keys(max_rows=150) == 200
    assert np.array_equal(np.sort(ctx.download_keys()), np.sort(pool[200:]))
    assert ctx.evict_keys(max_rows=100) == 0  # at the limit: nothing leaves
    assert ctx.evict_keys(max_rows=99) == 100  # all of age 0 tie
    assert len(ctx.download_keys()) == 0
    ctx.close()


# ---- 2. state ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["adagrad", "ftrl", "ps_adagrad"])
def test_survivors_keep_their_state_bit_for_bit(opt):
    cap = 4000
    batches = history(5, n_up=8)
    ctx = _ctx("fm", cap, OPTS[opt])
    replay(ctx, batches, train=True)
    table = ctx.download_keys()
    n = len(table)
    before = _rows(ctx)
    keys, We, Ve = ctx.evict_keys(max_rows=n // 2, export=True)
    new = ctx.download_keys()
    n_live = len(new)
    assert n_live <= n // 2 and n_live + len(keys) == n
    pos = {k: i for i, k in enumerate(table.tolist())}
    old = np.array([pos[k] for k in new.tolist()])
    after = _rows(ctx)
    for a, b in zip(before, after):  # survivors by key
        assert np.array_equal(bits(b[:n_live]), bits(a[old]))
    ev = np.array([pos[k] for k in keys.tolist()])
    assert np.array_equal(bits(We), bits(before[0][ev]))
    assert np.array_equal(bits(Ve), bits(before[1][ev].ravel()))
    fresh = _ctx("fm", cap, OPTS[opt])
    for a, b in zip(after, _rows(fresh)):  # vacated rows as lctr_create leaves them
        assert np.array_equal(bits(a[n_live:]), bits(b[n_live:]))
    ctx.close(); fresh.close()


# ---- 3. training goes on -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("opt", ["adagrad", "ftrl"])
def test_training_after_eviction_matches_a_context_seeded_with_the_survivors(opt):
    from lightctr_b200 import capi
    cap, k = 4000, K_FM
    batches = history(8, n_up=8)
    a = _ctx("fm", cap, OPTS[opt])
    replay(a, batches, train=True)
    n = len(a.download_keys())
    gone, We, Ve = a.evict_keys(max_rows=n // 2, export=True)
    live = a.download_keys()
    n_live = len(live)
    W, V = a.download_params()
    s1, s2 = a.download_opt_state()
    b = capi.Context(capi.MODEL_FM, cap, k, optimizer=OPTS[opt], key_mode=capi.KEYS_HASHED)
    b.upload_keyed_params(live, W[:n_live], V[:n_live * k])
    assert np.array_equal(b.lookup_keys(live), np.arange(n_live))
    b.upload_opt_state(s1, s2 if opt == "ftrl" else None)
    # the last batch with a tenth of its entries replaced by evicted keys, which come back as new keys
    rng = np.random.default_rng(3)
    last = batches[-1]
    keys = last.keys.copy()
    back = rng.random(len(keys)) < 0.1
    keys[back] = gone[rng.integers(0, len(gone), int(back.sum()))]
    bt = Batch(keys, 6, rng)
    bt.upload(a, 0)
    bt.upload(b, 0)
    ret = np.unique(keys[back])
    ra = a.lookup_keys(ret)
    assert np.all(ra >= n_live)
    Wa, Va = a.download_params()
    s1a, s2a = a.download_opt_state()
    assert np.all(Wa[ra] == 0)
    assert np.max(np.abs(Va.reshape(cap, k)[ra] - init_v(ret, k, 0, 1.0 / np.sqrt(k)))) < 1e-6
    assert np.all(s1a[ra] == 0) and np.all(s1a[cap:].reshape(cap, k)[ra] == 0)
    assert np.all(s2a[ra] == 0)
    la, lb = a.train_step(0)[0], b.train_step(0)[0]
    assert abs(la - lb) <= 1e-6 * abs(lb), (la, lb)
    allk = a.download_keys()
    ra, rb = a.lookup_keys(allk), b.lookup_keys(allk)
    Wa, Va = a.download_params()
    Wb, Vb = b.download_params()
    assert np.max(np.abs(Wa[ra] - Wb[rb])) < 2e-5
    assert np.max(np.abs(Va.reshape(cap, k)[ra] - Vb.reshape(cap, k)[rb])) < 2e-5
    # exported rows re-uploaded come back bit for bit
    a.upload_keyed_params(gone, We, Ve)
    rg = a.lookup_keys(gone)
    Wa, Va = a.download_params()
    assert np.array_equal(bits(Wa[rg]), bits(We))
    assert np.array_equal(bits(Va.reshape(cap, k)[rg].ravel()), bits(Ve))
    a.close(); b.close()


# ---- 4. staleness --------------------------------------------------------------------------------------------------
def test_resident_slots_go_stale_only_when_rows_were_freed():
    from lightctr_b200 import capi
    batches = history(4, n_up=4)
    ctx = _ctx("fm", 4000)
    replay(ctx, batches)
    assert ctx.evict_keys(max_idle=100) == 0  # nothing freed: every slot stays usable
    ctx.train_step(3)
    ctx.predict(2)
    assert ctx.evict_keys(max_idle=1) > 0
    for s in range(4):
        with pytest.raises(capi.LctrError, match="stale"):
            ctx.train_step(s)
        with pytest.raises(capi.LctrError, match="stale"):
            ctx.predict(s)
    batches[3].upload(ctx, 3)
    ctx.train_step(3)
    assert np.all(np.isfinite(ctx.predict(3)))
    ctx.close()


# ---- 5. a key stream larger than the capacity ----------------------------------------------------------------------
def _drift(n_batches, seed=9, rows=100, per=5, window=600, shift=200):
    rng = np.random.default_rng(seed)
    pool = fmix64(np.arange(window + shift * n_batches, dtype=np.uint64) + np.uint64(1 << 45))
    return [Batch(pool[i * shift + rng.integers(0, window, rows * per)], per, rng) for i in range(n_batches)]


def test_drifting_stream_past_the_capacity():
    cap, NB = 2000, 24
    batches = _drift(NB)
    seen, fail_at = set(), None
    for i, b in enumerate(batches):
        seen |= set(b.keys.tolist())
        if len(seen) > cap and fail_at is None:
            fail_at = i
    assert fail_at is not None and fail_at < 12
    assert len(seen) > 2 * cap
    # without eviction: the predicted batch fails
    plain = _ctx("fm", cap, key_evict=False)
    for i in range(fail_at):
        batches[i].upload(plain, 0)
        plain.train_step(0)
    from lightctr_b200 import capi
    with pytest.raises(capi.LctrError, match="capacity of %d rows" % cap):
        batches[fail_at].upload(plain, 0)
    plain.close()
    # with eviction before each upload: room for every key of the batch
    ctx = _ctx("fm", cap)
    losses = []
    for b in batches:
        ctx.evict_keys(max_rows=cap - len(np.unique(b.keys)))
        b.upload(ctx, 0)
        losses.append(ctx.train_step(0)[0])
        assert len(ctx.download_keys()) <= cap
    assert len(losses) == NB and np.all(np.isfinite(losses))
    ctx.close()


def test_one_eviction_clears_the_keys_left_without_a_row():
    from lightctr_b200 import capi
    cap = 2000
    batches = _drift(12)
    ctx = _ctx("fm", cap)
    failed = None
    for i, b in enumerate(batches):
        try:
            b.upload(ctx, 0)
        except capi.LctrError as e:
            assert "capacity" in str(e)
            failed = i
            break
    assert failed is not None
    with pytest.raises(capi.LctrError, match="capacity"):  # its row-less keys fail it again
        batches[failed].upload(ctx, 0)
    assert ctx.evict_keys(max_rows=cap - len(np.unique(batches[failed].keys))) > 0
    batches[failed].upload(ctx, 0)
    assert np.all(ctx.lookup_keys(batches[failed].keys) >= 0)
    assert np.isfinite(ctx.train_step(0)[0])
    ctx.close()


# ---- 6. checkpoint -------------------------------------------------------------------------------------------------
def test_checkpoint_keeps_clock_and_stamps(tmp_path):
    from lightctr_b200 import capi
    cap = 4000
    batches = history(21, n_up=7)
    a = _ctx("fm", cap, OPTS["ftrl"])
    replay(a, batches, train=True)
    path = str(tmp_path / "tracked.ckpt")
    a.save_checkpoint(path)
    b = _ctx("fm", cap, OPTS["ftrl"])
    b.load_checkpoint(path)
    ka, Wa, Va = a.evict_keys(max_idle=2, export=True)
    kb, Wb, Vb = b.evict_keys(max_idle=2, export=True)
    assert len(ka) > 0
    assert np.array_equal(ka, kb) and np.array_equal(bits(Wa), bits(Wb)) and np.array_equal(bits(Va), bits(Vb))
    assert np.array_equal(a.download_keys(), b.download_keys())
    for x, y in zip(_rows(a), _rows(b)):
        assert np.array_equal(bits(x), bits(y))
    # the clock goes on from the restored value
    for c in (a, b):
        batches[0].upload(c, 0)
    assert a.evict_keys(max_idle=0) == b.evict_keys(max_idle=0) > 0
    # keys new to that upload took rows in arrival order, which differs between the two: compare as sets
    assert np.array_equal(np.sort(a.download_keys()), np.sort(b.download_keys()))
    n = len(b.download_keys())
    b.save_checkpoint(path)
    # an untracked keyed checkpoint has exactly the layout it had before key_evict existed
    u = _ctx("fm", cap, OPTS["ftrl"], key_evict=False)
    replay(u, batches, train=True)
    upath = str(tmp_path / "untracked.ckpt")
    u.save_checkpoint(upath)
    F, r, nu = cap + 1, K_FM, len(u.download_keys())
    header = 8 + 4 * 4 + 5 * 8 + 2 * 9 * 4
    tables = 4 * F * (1 + r) * 3  # W, V | s1W, s1V | s2W, s2V
    assert os.path.getsize(upath) == header + tables + 8 + 8 * nu
    assert os.path.getsize(path) == header + tables + 8 + 8 * n + 8 + 8 * n  # + clock + stamps
    with pytest.raises(capi.LctrError, match="different trainer"):
        u.load_checkpoint(path)
    with pytest.raises(capi.LctrError, match="different trainer"):
        b.load_checkpoint(upath)
    a.close(); b.close(); u.close()


# ---- 7. rejections and memory --------------------------------------------------------------------------------------
def test_rejections_and_device_bytes():
    from lightctr_b200 import capi
    dense = capi.Context(capi.MODEL_FM, 1000, 8)
    with pytest.raises(capi.LctrError, match="key_mode"):
        dense.evict_keys(max_idle=0)
    with pytest.raises(capi.LctrError, match="key_evict"):
        capi.Context(capi.MODEL_FM, 1000, 8, key_evict=True)
    untracked = _ctx("fm", 1000, key_evict=False)
    with pytest.raises(capi.LctrError, match="key_evict"):
        untracked.evict_keys(max_idle=0)
    cap = 100000
    t = _ctx("fm", cap)
    u = _ctx("fm", cap, key_evict=False)
    assert t.device_bytes()[0] - u.device_bytes()[0] == cap * 8
    t.close(); u.close(); dense.close(); untracked.close()


def test_too_small_export_changes_nothing():
    from lightctr_b200 import capi
    batches = history(31, n_up=4)
    ctx = _ctx("fm", 4000)
    replay(ctx, batches, train=True)
    table = ctx.download_keys()
    before = _rows(ctx)
    keys = np.zeros(1, np.uint64)
    n = C.c_uint64()
    rc = ctx.L.lctr_evict_keys(ctx.h, 0, capi.NO_LIMIT, keys.ctypes.data, None, None, 1, C.byref(n))
    assert rc != 0 and "room for 1" in capi.load_library().lctr_last_error().decode()
    assert np.array_equal(ctx.download_keys(), table)
    for x, y in zip(before, _rows(ctx)):
        assert np.array_equal(bits(x), bits(y))
    ctx.train_step(3)  # slots stay usable
    assert ctx.evict_keys(max_idle=0) > 0
    ctx.close()
