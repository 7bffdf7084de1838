"""Keyed mode (cfg.key_mode = LCTR_KEYS_HASHED, csrc/keys.cu): batches carry 64-bit hashed keys, the library maps them to
table rows and creates + initialises rows on first sight.  After translation a slot holds ordinary row ids, so a keyed
context seeded to rows == fids must train exactly like a dense one (held to the dense tests' per-step oracle parity),
lazily created rows must hold the documented generator's values whatever order keys arrive in, and the capacity, unseen
keys, checkpoints and refused calls behave as include/lightctr_b200.h states."""
import numpy as np
import pytest

from keyed_model import OPTS, init_v
from lightctr_b200.dist import fmix64

pytestmark = pytest.mark.gpu


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-30)


def _synth(F, B, seed):
    from lightctr_b200.data import CriteoSynth
    return CriteoSynth(F, seed=seed).batch(B)


def _params_close(got, want, tol, threshold_updater):
    d = np.abs(got - want)
    if not threshold_updater:
        return float(d.max()) < tol
    return float(np.mean(d > tol)) <= 1e-5 and float(d.max()) < 1e-2


@pytest.mark.parametrize("opt", ["adagrad", "ftrl", "ps_adagrad"])
@pytest.mark.parametrize("k", [8, 16])
def test_keyed_fm_equals_dense_vs_oracle(oracle_api, opt, k):
    """keys = fmix64(fid) seeded in fid order -> row == fid; three steps, each from the oracle's state, at the dense
    fused-path bar (test_fused_step_vs_oracle: 1e-6 on the summed loss)"""
    from lightctr_b200 import capi
    F, B = 20000, 700
    rp, fid, fld, lab = _synth(F, B, 5 + k)
    rng = np.random.default_rng(k)
    W0 = (rng.standard_normal(F) * 0.01).astype(np.float32)
    V0 = (rng.standard_normal(F * k) / np.sqrt(k)).astype(np.float32) * np.float32(0.5)
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, 0)
    o = oracle_api.FMOracle(ds, k, W0, V0)
    o.opt = opt
    ctx = capi.Context(capi.MODEL_FM, F, k, optimizer=OPTS[opt], deterministic=0, key_mode=capi.KEYS_HASHED)
    ctx.upload_keyed_params(fmix64(np.arange(F)), W0, V0)
    keys = fmix64(fid)
    assert np.array_equal(ctx.lookup_keys(keys), fid.astype(np.int64))
    ctx.upload_batch_keys(0, rp, keys, None, None, lab)
    F1 = F * (k + 1)
    for step in range(3):
        if step > 0:
            ctx.upload_params(o.W, o.V)
            ctx.upload_opt_state(o.accum, getattr(o, "s2", np.zeros(F1, np.float32)) if opt == "ftrl" else None)
        lg, cg = ctx.train_step(0)
        lo, ao = o.epoch()
        assert _rel(lg, lo) < 1e-6, (opt, k, step, lg, lo)
        assert abs(cg - round(ao * B)) <= 1
        Wg, Vg = ctx.download_params()
        thr = opt == "ftrl"
        assert _params_close(Wg, o.W, 2e-5, thr) and _params_close(Vg, o.V, 2e-5, thr), (opt, k, step)
    assert np.array_equal(ctx.download_keys(), fmix64(np.arange(F)))
    ctx.close()


def test_keyed_ffm_equals_dense_vs_oracle(oracle_api):
    """FFM k = 4 on a keyed context seeded to rows == fids: the dense FFM bar (1e-5 on the loss, 2e-5 on parameters)"""
    from lightctr_b200 import capi
    F, B, Fc, k = 5000, 400, 39, 4
    rp, fid, fld, lab = _synth(F, B, 21)
    rng = np.random.default_rng(3)
    W0 = (rng.standard_normal(F) * 0.05).astype(np.float32)
    V0 = (rng.standard_normal(F * Fc * k) * 0.1).astype(np.float32)
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, Fc)
    o = oracle_api.FFMOracle(ds, k, W0, V0)
    ctx = capi.Context(capi.MODEL_FFM, F, k, Fc, deterministic=0, key_mode=capi.KEYS_HASHED)
    ctx.upload_keyed_params(fmix64(np.arange(F)), W0, V0)
    keys = fmix64(fid)
    assert np.array_equal(ctx.lookup_keys(keys), fid.astype(np.int64))
    ctx.upload_batch_keys(0, rp, keys, fld, None, lab)
    for step in range(3):
        lg, cg = ctx.train_step(0)
        lo, ao = o.epoch()
        assert _rel(lg, lo) < 1e-5, (step, lg, lo)
        assert abs(cg - round(ao * B)) <= 1
        Wg, Vg = ctx.download_params()
        assert np.max(np.abs(Wg - o.W)) < 2e-5 and np.max(np.abs(Vg - o.V)) < 2e-5
        ctx.upload_params(o.W, o.V)
        ctx.upload_opt_state(o.s1)
    ctx.close()


def test_keyed_nfm_equals_dense_vs_oracle(oracle_api):
    """NFM k = 16, fp32 chain 16 -> 64 -> 32 -> 1, one minibatch per step: the first step against the oracle at the dense NFM
    bar (1e-5, as test_c4_shape_nfm_chain_fp32_one_step: the oracle re-draws its dropout masks after a step), then three
    steps against a dense context seeded alike (the same kernels; 2e-5, the order-free path's own reproducibility)"""
    from lightctr_b200 import capi
    F, B, k = 20000, 2048, 16
    hidden = [64, 32]
    rp, fid, fld, lab = _synth(F, B, 44)
    rng = np.random.default_rng(4)
    W0 = (rng.standard_normal(F) * 0.01).astype(np.float32)
    V0 = (rng.standard_normal(F * k, dtype=np.float32) * np.float32(0.25))
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, 0)
    o = oracle_api.NFMOracle(ds, k, hidden, W=W0, V=V0, batch_size=B, minibatch=B)
    dims = [k] + hidden + [1]
    ctx = capi.Context(capi.MODEL_NFM, F, k, hidden=tuple(hidden), mlp_precision=capi.MLP_FP32, minibatch_size=B,
                       deterministic=0, key_mode=capi.KEYS_HASHED)
    dense = capi.Context(capi.MODEL_NFM, F, k, hidden=tuple(hidden), mlp_precision=capi.MLP_FP32, minibatch_size=B,
                         deterministic=0)
    for l in range(len(dims) - 1):
        w = ((rng.random(dims[l] * dims[l + 1], dtype=np.float32) - np.float32(0.5)) * np.float32(2.0 / np.sqrt(dims[l])))
        o.mlp.arrays("weight", l)[:] = w
        o.mlp.arrays("bias", l)[:] = 0
        o.mlp.arrays("mask", l)[:] = 1.0
        ctx.mlp_upload(l, w, np.zeros(dims[l + 1], np.float32))
        dense.mlp_upload(l, w, np.zeros(dims[l + 1], np.float32))
    ctx.upload_keyed_params(fmix64(np.arange(F)), W0, V0)
    ctx.upload_batch_keys(0, rp, fmix64(fid), None, None, lab)
    dense.upload_params(W0, V0)
    dense.upload_batch(0, rp, fid, None, None, lab)
    lg, _ = ctx.train_step(0)
    lo, _ = o.epoch()
    assert _rel(lg, lo) < 1e-5, (lg, lo)
    Wg, Vg = ctx.download_params()
    assert np.max(np.abs(Wg - o.W)) < 1e-4
    assert float(np.mean(np.abs(Vg - o.V) > 1e-4)) <= 1e-5
    ld = dense.train_step(0)[0]
    assert _rel(lg, ld) < 1e-6, (lg, ld)
    for step in range(3):
        lg, ld = ctx.train_step(0)[0], dense.train_step(0)[0]
        assert _rel(lg, ld) < 2e-5, (step, lg, ld)
    ctx.close(); dense.close()


@pytest.mark.parametrize("opt", ["adagrad", "ps_adagrad", "ftrl"])
def test_lazy_init_and_order_independence(opt):
    from lightctr_b200 import capi
    F, k, B = 50000, 16, 1500
    salt = np.uint64(0x5bd1e995)
    batches = []
    for i in range(3):
        rp, fid, fld, lab = _synth(F, B, 60 + i)
        batches.append((rp, fmix64(fid.astype(np.uint64) ^ salt), lab))
    ukeys = np.unique(np.concatenate([b[1] for b in batches]))
    U = len(ukeys)
    seed, scale = 77, 0.3
    maps = []
    for order in ((0, 1, 2), (2, 0, 1)):
        ctx = capi.Context(capi.MODEL_FM, 2 * U, k, optimizer=OPTS[opt], key_mode=capi.KEYS_HASHED)
        ctx.set_key_init(seed, scale)
        for slot, i in enumerate(order):
            rp, keys, lab = batches[i]
            ctx.upload_batch_keys(slot, rp, keys, None, None, lab)
        rows = ctx.lookup_keys(ukeys)
        assert len(np.unique(rows)) == U and rows.min() == 0 and rows.max() == U - 1
        table = ctx.download_keys()
        assert len(table) == U and np.array_equal(table[rows], ukeys)
        W, V = ctx.download_params()
        V = V.reshape(-1, k)
        assert np.all(W == 0)
        assert np.max(np.abs(V[rows] - init_v(ukeys, k, seed, scale))) < 1e-6
        assert np.all(V[U:] == 0)  # rows not allocated read as zero
        s1, s2 = ctx.download_opt_state()
        want = np.float32(1e-7) if opt == "ps_adagrad" else np.float32(0)
        s1W, s1V = s1[:2 * U], s1[2 * U:].reshape(-1, k)
        assert np.all(s1W[:U] == want) and np.all(s1V[:U] == want)
        if opt == "ftrl":
            assert np.all(s2 == 0)
        maps.append((W[rows].copy(), V[rows].copy()))
        ctx.close()
    # same key -> bit-identical (W, V) whatever order the batches came in
    assert np.array_equal(maps[0][0].view(np.uint32), maps[1][0].view(np.uint32))
    assert np.array_equal(maps[0][1].view(np.uint32), maps[1][1].view(np.uint32))


def test_default_init_scale_is_inverse_sqrt_k():
    from lightctr_b200 import capi
    k = 8
    ctx = capi.Context(capi.MODEL_FM, 100, k, key_mode=capi.KEYS_HASHED)
    keys = fmix64(np.arange(10) + 1000)
    ctx.upload_batch_keys(0, np.array([0, 10]), keys, None, None, np.array([1]))
    _, V = ctx.download_params()
    rows = ctx.lookup_keys(keys)
    assert np.max(np.abs(V.reshape(-1, k)[rows] - init_v(keys, k, 0, 1.0 / np.sqrt(k)))) < 1e-6
    ctx.close()


def test_free_run_matches_dense_context_seeded_from_keyed_download():
    from lightctr_b200 import capi
    F, k, B, NB = 40000, 16, 1024, 3
    batches = []
    for i in range(NB):
        rp, fid, fld, lab = _synth(F, B, 200 + i)
        batches.append((rp, fmix64(fid.astype(np.uint64) + np.uint64(1 << 40)), lab))
    cap = 30000
    a = capi.Context(capi.MODEL_FM, cap, k, key_mode=capi.KEYS_HASHED)
    for i, (rp, keys, lab) in enumerate(batches):
        a.upload_batch_keys(i, rp, keys, None, None, lab)
    W, V = a.download_params()
    b = capi.Context(capi.MODEL_FM, cap, k)
    b.upload_params(W, V)
    for i, (rp, keys, lab) in enumerate(batches):
        b.upload_batch(i, rp, a.lookup_keys(keys).astype(np.uint32), None, None, lab)
    la = [a.train_step(s % NB)[0] for s in range(10)]
    lb = [b.train_step(s % NB)[0] for s in range(10)]
    la, lb = np.array(la), np.array(lb)
    assert np.max(np.abs(la - lb) / np.abs(lb)) < 2e-5, np.max(np.abs(la - lb) / np.abs(lb))
    a.close(); b.close()


def test_capacity_overflow_is_an_error_that_keeps_the_table():
    from lightctr_b200 import capi
    k, B = 8, 300
    rp, fid, fld, lab = _synth(5000, B, 9)
    keys = fmix64(fid.astype(np.uint64) + np.uint64(7))
    U = len(np.unique(keys))
    ctx = capi.Context(capi.MODEL_FM, U, k, key_mode=capi.KEYS_HASHED)
    ctx.upload_batch_keys(0, rp, keys, None, None, lab)
    ctx.train_step(0)
    table = ctx.download_keys()
    assert len(table) == U
    W0, V0 = ctx.download_params()
    keys2 = keys.copy()
    keys2[5] = np.uint64(123456789)  # one key the table has not seen
    for _ in range(2):  # a later upload meeting the row-less key fails the same way
        with pytest.raises(capi.LctrError, match="capacity of %d rows" % U):
            ctx.upload_batch_keys(1, rp, keys2, None, None, lab)
        assert np.array_equal(ctx.download_keys(), table)
        with pytest.raises(capi.LctrError, match="no usable batch"):
            ctx.train_step(1, 0, B)
    W1, V1 = ctx.download_params()
    assert np.array_equal(W0, W1) and np.array_equal(V0, V1)
    assert ctx.lookup_keys(keys2[5:6])[0] == -1
    ctx.upload_batch_keys(1, rp, keys2, None, None, lab, insert=False)  # lookup only: predicts normally
    p = ctx.predict(1)
    assert p.shape == (B,) and np.all(np.isfinite(p)) and np.all((p > 0) & (p < 1))
    with pytest.raises(capi.LctrError, match="insert = 0"):
        ctx.train_step(1)
    ctx.train_step(0)  # the slot that was uploaded before still trains
    ctx.close()


def test_unseen_keys_predict_as_dropped_features():
    from lightctr_b200 import capi
    F, k, B = 20000, 16, 800
    rp, fid, fld, lab = _synth(F, B, 13)
    keys = fmix64(fid.astype(np.uint64))
    # small parameters (init scale 0.1, lr 0.01) keep the FM interaction's cancellation noise -- the two predictions sum a
    # row's terms in different orders -- well below the 1e-6 bar on pCTR
    ctx = capi.Context(capi.MODEL_FM, 30000, k, lr=0.01, key_mode=capi.KEYS_HASHED)
    ctx.set_key_init(0, 0.1)
    ctx.upload_batch_keys(0, rp, keys, None, None, lab)
    for _ in range(3):
        ctx.train_step(0)
    n_rows = len(ctx.download_keys())
    # test batch: every entry but the first of each row replaced by an unseen key with probability 0.3
    rng = np.random.default_rng(1)
    tkeys = keys.copy()
    unseen = rng.random(len(keys)) < 0.3
    unseen[rp[:-1]] = False
    tkeys[unseen] = fmix64(np.arange(unseen.sum(), dtype=np.uint64) + np.uint64(1 << 50))
    assert np.all(ctx.lookup_keys(tkeys[unseen]) == -1)
    ctx.upload_batch_keys(1, rp, tkeys, None, None, lab, insert=False)
    p_keyed = ctx.predict(1)
    assert len(ctx.download_keys()) == n_rows
    W, V = ctx.download_params()
    d = capi.Context(capi.MODEL_FM, 30000, k, lr=0.01)
    d.upload_params(W, V)
    keep = ~unseen
    counts = np.add.reduceat(keep.astype(np.int64), rp[:-1])
    rp2 = np.concatenate([[0], np.cumsum(counts)]).astype(np.int64)
    d.upload_batch(0, rp2, ctx.lookup_keys(keys[keep]).astype(np.uint32), None, None, lab)
    p_dense = d.predict(0)
    assert np.max(np.abs(p_keyed - p_dense)) < 1e-6, np.max(np.abs(p_keyed - p_dense))
    ctx.close(); d.close()


def test_checkpoint_roundtrip_rebuilds_the_table(tmp_path):
    from lightctr_b200 import capi
    F, k, B = 20000, 8, 600
    rp, fid, fld, lab = _synth(F, B, 17)
    keys = fmix64(fid.astype(np.uint64) * np.uint64(3))
    cap = 25000
    a = capi.Context(capi.MODEL_FM, cap, k, optimizer=capi.OPT_FTRL, key_mode=capi.KEYS_HASHED)
    a.upload_batch_keys(0, rp, keys, None, None, lab)
    for _ in range(3):
        a.train_step(0)
    path = str(tmp_path / "keyed.ckpt")
    a.save_checkpoint(path)
    b = capi.Context(capi.MODEL_FM, cap, k, optimizer=capi.OPT_FTRL, key_mode=capi.KEYS_HASHED)
    b.load_checkpoint(path)
    ka, kb = a.download_keys(), b.download_keys()
    assert np.array_equal(ka, kb)
    for x, y in zip(a.download_params() + a.download_opt_state(), b.download_params() + b.download_opt_state()):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))
    assert np.array_equal(a.lookup_keys(ka), b.lookup_keys(ka))
    assert np.array_equal(b.lookup_keys(ka), np.arange(len(ka)))
    b.upload_batch_keys(0, rp, keys, None, None, lab)  # and training goes on from the restored table
    assert _rel(b.train_step(0)[0], a.train_step(0)[0]) < 1e-5
    dense = capi.Context(capi.MODEL_FM, cap + 1, k, optimizer=capi.OPT_FTRL)
    with pytest.raises(capi.LctrError, match="different trainer"):
        dense.load_checkpoint(path)
    a.close(); b.close(); dense.close()


def test_rejections():
    from lightctr_b200 import capi
    with pytest.raises(capi.LctrError, match="single-GPU"):
        capi.Context(capi.MODEL_FM, 1000, 8, world=2, rank=0, key_mode=capi.KEYS_HASHED)
    with pytest.raises(capi.LctrError, match="deterministic"):
        capi.Context(capi.MODEL_FM, 1000, 8, deterministic=1, key_mode=capi.KEYS_HASHED)
    with pytest.raises(capi.LctrError, match="deterministic"):
        capi.Context(capi.MODEL_FM, 1000, 8, deterministic=2, key_mode=capi.KEYS_HASHED)
    ctx = capi.Context(capi.MODEL_FM, 1000, 8, key_mode=capi.KEYS_HASHED)
    rp = np.array([0, 2, 3], np.int64)
    lab = np.array([1, 0], np.int32)
    with pytest.raises(capi.LctrError, match="reserved"):
        ctx.upload_batch_keys(0, rp, np.array([5, capi.RESERVED_KEY, 9], np.uint64), None, None, lab)
    with pytest.raises(capi.LctrError, match="reserved"):
        ctx.upload_keyed_params(np.array([capi.RESERVED_KEY], np.uint64), np.zeros(1, np.float32))
    with pytest.raises(capi.LctrError, match="more than once"):
        ctx.upload_keyed_params(np.array([4, 4], np.uint64), np.zeros(2, np.float32))
    assert len(ctx.download_keys()) == 0
    fid = np.array([1, 2, 3], np.uint32)
    with pytest.raises(capi.LctrError, match="lctr_upload_batch_keys"):
        ctx.upload_batch(0, rp, fid, None, None, lab)
    with pytest.raises(capi.LctrError, match="keyed"):
        ctx.train_batch(rp, fid, None, None, lab)
    with pytest.raises(capi.LctrError, match="keyed"):
        ctx.train_batch_async(rp, fid, None, None, lab)
    dense = capi.Context(capi.MODEL_FM, 1000, 8)
    with pytest.raises(capi.LctrError, match="key_mode"):
        dense.upload_batch_keys(0, rp, np.array([5, 6, 9], np.uint64), None, None, lab)
    ctx.close(); dense.close()


def test_device_bytes_count_the_key_table():
    from lightctr_b200 import capi
    cap, k = 100000, 16
    a = capi.Context(capi.MODEL_FM, cap, k, key_mode=capi.KEYS_HASHED)
    d = capi.Context(capi.MODEL_FM, cap + 1, k)
    T = 1 << int(np.ceil(np.log2(2 * cap)))
    assert a.device_bytes()[0] - d.device_bytes()[0] == T * 12 + cap * 8
    a.close(); d.close()
