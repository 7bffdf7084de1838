"""Single-GPU checkpoints (csrc/checkpoint.cu).  The saved bytes must equal the documented layout built with numpy from the
context's own downloads; a keyed load must make resident keyed slots stale; and a refused load must leave every download
as it was."""
import struct

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

MAX_LAYERS = 8
TWO_STATE = {1, 2, 4, 7, 8}  # FTRL, Adam, Adadelta, PS DCASGD, PS DCASGDA keep s2 beside s1


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _batch(seed, F, rows=256, per=10, Fc=0):
    rng = np.random.default_rng(seed)
    rp = np.arange(0, rows * per + 1, per, dtype=np.int64)
    fid = rng.integers(0, F, rows * per).astype(np.uint32)
    field = (fid % Fc).astype(np.uint16) if Fc else None
    lab = (rng.random(rows) < 0.3).astype(np.int32)
    return rp, fid, field, lab


def _keys(fid):
    from lightctr_b200 import dist as ldist
    return ldist.fmix64(fid.astype(np.uint64) + np.uint64(1))


def _expected(ctx, step, layers=(), adam_iter=0, clock=None, stamps=None):
    """the file lctr_save_checkpoint writes for a single-GPU context: the 136-byte header, W, V, s1W, s1V[, s2W, s2V] over
    every row, then per layer w, b, acc_w, acc_b, mask, then (keyed) the row count and keys, (key_evict = 1) the clock and
    stamps.  `layers`: (in, out, w, b, acc_w, acc_b, mask) per layer."""
    cfg = ctx.cfg
    keyed = cfg.key_mode != 0
    F = ctx.F + (1 if keyed else 0)  # keyed tables keep the null row of unseen keys after the capacity
    dims = [(l[0], l[1]) for l in layers] + [(0, 0)] * (MAX_LAYERS + 1 - len(layers))
    out = [b"LCTRCKP1", struct.pack("<4i", cfg.model, cfg.optimizer, len(layers), cfg.key_mode | (0x100 if cfg.key_evict else 0)),
           struct.pack("<5Q", F, cfg.field_cnt, cfg.factor_cnt, adam_iter, step),
           struct.pack("<%di" % (MAX_LAYERS + 1), *[d[0] for d in dims]),
           struct.pack("<%di" % (MAX_LAYERS + 1), *[d[1] for d in dims])]
    assert sum(len(x) for x in out) == 136
    W, V = ctx.download_params()
    s1, s2 = ctx.download_opt_state()
    n = ctx.F
    sections = [W, V, s1[:n], s1[n:]] + ([s2[:n], s2[n:]] if cfg.optimizer in TWO_STATE else [])
    for a, sec in enumerate(sections):
        out.append(np.ascontiguousarray(sec, np.float32).tobytes())
        if keyed:  # the null row: never trained, in the state lctr_create gives (s1 = 0 for the rules used here)
            out.append(np.zeros(ctx.rowlen if a % 2 else 1, np.float32).tobytes())
    for l in layers:
        out += [np.ascontiguousarray(x, np.float32).tobytes() for x in l[2:]]
    if keyed:
        keys = ctx.download_keys()
        out += [struct.pack("<Q", len(keys)), keys.astype("<u8").tobytes()]
        if cfg.key_evict:
            out += [struct.pack("<Q", clock), np.asarray(stamps, "<u8").tobytes()]
    return b"".join(out)


def _fm_adagrad(capi):
    F, k = 5000, 8
    c = capi.Context(capi.MODEL_FM, F, k, optimizer=capi.OPT_ADAGRAD)
    rp, fid, _, lab = _batch(1, F)
    c.upload_batch(0, rp, fid, None, None, lab)
    for _ in range(3):
        c.train_step(0)
    return c, dict(step=3)


def _ffm_ftrl(capi):
    F, k, Fc = 2000, 4, 5
    c = capi.Context(capi.MODEL_FFM, F, k, Fc, optimizer=capi.OPT_FTRL)
    rp, fid, field, lab = _batch(2, F, Fc=Fc)
    c.upload_batch(0, rp, fid, field, None, lab)
    for _ in range(2):
        c.train_step(0)
    return c, dict(step=2)


def _keyed_fm(capi, key_evict):
    cap, k = 3000, 8
    c = capi.Context(capi.MODEL_FM, cap, k, optimizer=capi.OPT_ADAGRAD, key_mode=capi.KEYS_HASHED, key_evict=key_evict)
    met = []
    for i, lo in enumerate((0, 600)):  # two insert-uploads over overlapping key ranges: clock 1, then 2
        rp, fid, _, lab = _batch(3 + i, 1000)
        keys = _keys(fid + lo)
        c.upload_batch_keys(0, rp, keys, None, None, lab)
        c.train_step(0)
        met.append(set(keys.tolist()))
    stamps = [2 if key in met[1] else 1 for key in c.download_keys().tolist()]
    return c, dict(step=2, clock=2, stamps=stamps)


def _nfm_masked(capi):
    F, k, H = 3000, 8, 32
    c = capi.Context(capi.MODEL_NFM, F, k, hidden=(H,), minibatch_size=256)
    rng = np.random.default_rng(4)
    c.upload_params((rng.standard_normal(F) * 0.01).astype(np.float32), (rng.standard_normal(F * k) / 4).astype(np.float32))
    layers = []
    for l, (i, o) in enumerate(((k, H), (H, 1))):
        w, b = (rng.random(i * o, dtype=np.float32) - 0.5), rng.random(o, dtype=np.float32)
        mask = (rng.random(o) < 0.7).astype(np.float32) if l == 0 else np.ones(o, np.float32)
        c.mlp_upload(l, w, b)
        c.mlp_set_mask(l, mask)
        layers.append((i, o, w, b, np.zeros(i * o, np.float32), np.zeros(o, np.float32), mask))
    return c, dict(step=0, layers=layers)


CASES = {
    "fm_adagrad": _fm_adagrad,
    "ffm_ftrl": _ffm_ftrl,
    "keyed_fm": lambda capi: _keyed_fm(capi, False),
    "keyed_fm_tracked": lambda capi: _keyed_fm(capi, True),
    "nfm_masked_layers": _nfm_masked,
}


@pytest.mark.parametrize("case", list(CASES))
def test_saved_bytes_follow_the_documented_layout(tmp_path, case):
    from lightctr_b200 import capi
    c, kw = CASES[case](capi)
    path = str(tmp_path / "ckpt")
    c.save_checkpoint(path)
    got, want = open(path, "rb").read(), _expected(c, **kw)
    c.close()
    assert len(got) == len(want), (len(got), len(want))
    diff = np.nonzero(np.frombuffer(got, np.uint8) != np.frombuffer(want, np.uint8))[0]
    assert len(diff) == 0, "first differing byte at offset %d" % diff[0]


def _keyed_ftrl(capi, cap=3000):
    return capi.Context(capi.MODEL_FM, cap, 8, optimizer=capi.OPT_FTRL, key_mode=capi.KEYS_HASHED)


def test_single_gpu_keyed_load_makes_resident_slots_stale(tmp_path):
    from lightctr_b200 import capi
    rp, fid, _, lab = _batch(5, 1000)
    a = _keyed_ftrl(capi)
    a.upload_batch_keys(0, rp, _keys(fid), None, None, lab)
    a.train_step(0)
    path = str(tmp_path / "keyed")
    a.save_checkpoint(path)
    a.close()
    b = _keyed_ftrl(capi)
    rp2, fid2, _, lab2 = _batch(6, 1000)
    b.upload_batch_keys(0, rp2, _keys(fid2 + 500), None, None, lab2)  # translated under b's own numbering
    b.load_checkpoint(path)
    with pytest.raises(capi.LctrError, match="stale"):
        b.train_step(0)
    b.upload_batch_keys(0, rp2, _keys(fid2 + 500), None, None, lab2)
    assert np.isfinite(b.train_step(0)[0])
    b.close()


def test_refused_single_gpu_loads_change_nothing(tmp_path):
    from lightctr_b200 import capi
    cap = 3000
    src = _keyed_ftrl(capi, cap)
    rp, fid, _, lab = _batch(7, 1000)
    src.upload_batch_keys(0, rp, _keys(fid), None, None, lab)
    src.train_step(0)
    good = str(tmp_path / "good")
    src.save_checkpoint(good)
    n, rowlen = len(src.download_keys()), src.rowlen
    src.close()
    data = open(good, "rb").read()
    keys_at = len(data) - 8 * (1 + n)  # the row count, then the n keys
    too_many = _keys(np.arange(cap + 1, dtype=np.uint32) + np.uint32(10 ** 6))
    reserved = bytearray(data)
    reserved[keys_at + 8 + 8 * (n // 2):keys_at + 16 + 8 * (n // 2)] = b"\xff" * 8
    bad = {
        "cut inside V": data[:136 + 4 * (cap + 1) + 4 * (cap + 1) * rowlen // 2],
        "cut inside the keys": data[:len(data) - 8 * (n // 2)],
        "one trailing byte": data + b"\0",
        "reserved key": bytes(reserved),
        "rows above the capacity": data[:keys_at] + struct.pack("<Q", cap + 1) + too_many.astype("<u8").tobytes(),
    }

    c = _keyed_ftrl(capi, cap)
    rp2, fid2, _, lab2 = _batch(8, 1000)
    c.upload_batch_keys(0, rp2, _keys(fid2 + 300), None, None, lab2)
    c.train_step(0)
    for name, blob in bad.items():
        path = str(tmp_path / name.replace(" ", "_"))
        open(path, "wb").write(blob)
        before = c.download_params() + c.download_opt_state() + (c.download_keys(),)
        with pytest.raises(capi.LctrError):
            c.load_checkpoint(path)
        after = c.download_params() + c.download_opt_state() + (c.download_keys(),)
        for x, y in zip(before, after):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8)), name
        assert np.isfinite(c.train_step(0)[0]), name
    c.close()
