"""libffm text parsed into a slot on the device (lctr_upload_libffm) against the host loader: split at any line
boundaries, the slots hold bit for bit what lctr_load_libffm (+ lctr_upload_batch) gives on the whole text, parser quirks
included; keyed contexts match lctr_load_libffm_keys + lctr_upload_batch_keys; training from a text-uploaded slot
equals training from the host-parsed CSR."""
import os
import random

import numpy as np
import pytest

from golden_util import GOLDEN, load_csr, write_libffm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def capi():
    from lightctr_b200 import build as lbuild
    from lightctr_b200 import capi as _capi
    lbuild.build()
    _capi.load_library()
    return _capi


def _lines(text):
    """text split after every '\\n' (a last piece without one kept)"""
    out, pos = [], 0
    while pos < len(text):
        nl = text.find(b"\n", pos)
        end = len(text) if nl < 0 else nl + 1
        out.append(text[pos:end])
        pos = end
    return out


def _upload(ctx, parts, slot=0, lookup=False):
    """parts as consecutive calls -> concatenated (row_ptr, fid, field, val, label) of the slots, and the infos"""
    rp, fid, field, val, label, infos = [np.zeros(1, np.int64)], [], [], [], [], []
    base = 0
    for i, p in enumerate(parts):
        info = ctx.upload_libffm(slot, p, begin=i == 0, end=i == len(parts) - 1, lookup=lookup)
        assert info.consumed == len(p)
        r, f, fl, v, lb = ctx.download_batch(slot)
        assert r[0] == 0 and len(r) == info.rows + 1 and len(f) == info.nnz
        rp.append(r[1:] + base)
        base += int(r[-1])
        fid.append(f), field.append(fl), val.append(v), label.append(lb)
        infos.append(info)
    return [np.concatenate(a) for a in (rp, fid, field, val, label)], infos


def _reference(capi, text, tmp_path, keyed=False):
    p = str(tmp_path / "ref.txt")
    open(p, "wb").write(text)
    return capi.load_libffm_keys(p) if keyed else capi.load_libffm(p)


def _check_equal(got, ref):
    rp, fid, field, val, label = got
    assert np.array_equal(rp, ref.row_ptr)
    assert np.array_equal(fid, ref.fid)
    assert np.array_equal(field, ref.field)
    assert np.array_equal(val.view(np.uint32), ref.val.view(np.uint32))
    assert np.array_equal(label, ref.label[:ref.rows].astype(np.float32))


def _splits(text, rng, n_random=3):
    """the whole text, one line per call, a split after each featureless line, and random line-aligned splits"""
    lines = _lines(text)
    out = [[text], lines]
    cuts = [i + 1 for i, l in enumerate(lines[:-1]) if l.split(b"\t")[-1].strip() == b"" and l.strip()]
    if cuts:
        out.append([b"".join(lines[a:b]) for a, b in zip([0] + cuts, cuts + [len(lines)])])
    for _ in range(n_random):
        k = rng.randrange(1, max(2, min(len(lines), 6)))
        cut = sorted(rng.sample(range(1, len(lines)), k - 1)) if len(lines) > k else []
        out.append([b"".join(lines[a:b]) for a, b in zip([0] + cut, cut + [len(lines)])])
    return [[p for p in parts if p] or [b""] for parts in out]


def _dense(capi, F=1000, **kw):
    return capi.Context(capi.MODEL_FM, F, 4, **kw)


# ---- 1. golden data -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["train_sparse_csr.npz", "train_sparse_head.csv", "test_sparse_head.csv"])
def test_golden_text_equals_the_host_loader(capi, tmp_path, name):
    if name.endswith(".npz"):
        p = str(tmp_path / "train.txt")
        write_libffm(load_csr(name, field_cnt=68), p)
    else:
        p = os.path.join(GOLDEN, name)
    text = open(p, "rb").read()
    ref = capi.load_libffm(p)
    ctx = _dense(capi, F=int(ref.feature_cnt))
    for parts in _splits(text, random.Random(1), n_random=2):
        got, infos = _upload(ctx, parts)
        _check_equal(got, ref)
        assert sum(i.host_lines for i in infos) == 0
        assert sum(i.rows for i in infos) == ref.rows and sum(i.nnz for i in infos) == ref.nnz
        assert sum(i.labels for i in infos) == len(ref.label) and sum(i.lines for i in infos) == len(_lines(text))
        assert max(i.feature_cnt for i in infos) == ref.feature_cnt
        assert max(i.field_cnt for i in infos) == int(ref.field.max()) + 1
    assert all(i.host_lines == 0 for i in infos)


# ---- 2. quirks ----------------------------------------------------------------------------------------------------
# (text, the device grammar declines some line of it)
QUIRKS = [
    (b"1\t0:3:1 1:7:0.5\n1\t\n0\t5:9:1.25 6:10 7:12:3\n-1\t0:0:1e-3 1:1:-2.5\n", True),
    (b"1\t0:3:1 1:7:0.5\r\n0\t2:5:2\r\n\r\n1\t4:4:0.25\r\n", False),           # CRLF
    (b"1\t\t0:3:1   1:7:0.5\t\n0  2:5:2 \t 3:6:+1.5\n+1\t1:1:1\n", False),        # tabs, runs of spaces, + signs
    (b"1\t0:3:1e2 1:4:2\n0\t1:5:0x1p3\n1\t2:6:inf 3:7:nan\n0\t1:1:1E-2\n", True),  # exponents, hex floats, inf / nan
    (b"1\t0:0000000000000000012:1\n0\t1:5:1\n", True),                           # a 19-digit id
    (b"1234567890\t0:1:1\n12345678901\t1:2:1\n0\t3:3:1\n", True),                # 10- and 11-digit labels
    (b"1\t0:3:1\x00 1:4:1\n\x00\n0\t1:2:1\n", True),                              # NUL bytes
    (b"\n\n1\n0\t\n1\t0:1:0.5\n\n", False),                                      # empty and label-only lines
    (b"1\t0:3:1 junk 1:4:1\n0\t1:2:1 :\n", True),                                 # garbage after tokens
    (b"1\t0:3:2.5\n0\t1:4 2:5:1\n1\t3:6\n", True),                               # two-field token first on a line
    (b"1\t0:3:0.1 1:4:16777217 2:5:3.14159265358979\n0\t1:1:-0 2:2:.5 3:3:5.\n", True),  # a float midpoint
    (b"1\t0:3:1 1:4:0.5\n0\t2:5:2", False),                                      # no final newline
    (b"x\n1 0:1:1\n-\n0\t1:2:1", True),
]


@pytest.mark.parametrize("case", range(len(QUIRKS)))
def test_quirk_corpus_equals_the_host_loader(capi, tmp_path, case):
    text, declines = QUIRKS[case]
    ref = _reference(capi, text, tmp_path)
    ctx = _dense(capi)
    for parts in _splits(text, random.Random(case)):
        got, infos = _upload(ctx, parts)
        _check_equal(got, ref)
        assert (sum(i.host_lines for i in infos) > 0) == declines


def test_stale_value_carries_across_calls(capi, tmp_path):
    """a two-field token first on a line keeps the value of the last token before it, in an earlier call too"""
    text = b"1\t0:3:2.5\n1\t\n0\t1:4 2:5:1\n"
    ref = _reference(capi, text, tmp_path)
    assert ref.val[1] == np.float32(2.5) and ref.label.tolist() == [1, 1, 0] and ref.rows == 2
    got, _ = _upload(_dense(capi), _lines(text))
    _check_equal(got, ref)


def test_consumed_stops_at_the_last_newline(capi, tmp_path):
    ctx = _dense(capi)
    text = b"1\t0:3:1\n0\t1:4:0.5\n1\t2:5:2"
    info = ctx.upload_libffm(0, text, begin=True, end=False)
    assert info.consumed == text.rindex(b"\n") + 1 and info.rows == 2 and info.lines == 2
    info = ctx.upload_libffm(0, text[info.consumed:], begin=False, end=True)
    assert info.consumed == len(text) - text.rindex(b"\n") - 1 and info.rows == 1
    info = ctx.upload_libffm(0, b"1\t0:1:1", begin=True, end=False)
    assert info.consumed == 0 and info.rows == 0 and info.lines == 0


# ---- 3. seeded fuzz -----------------------------------------------------------------------------------------------
PIECES = [b"0:1:1e-3", b"1:2:0x10", b"2:3", b"junk", b"3:4:inf", b"00000000000000000007:1:1", b"4:5:1.00000000000000000001",
          b"5:6:-", b":", b"6:7:+2", b"\x00", b"7:8:33554433"]


def _fuzz_doc(rng):
    lines = []
    for _ in range(rng.randrange(1, 40)):
        r = rng.random()
        if r < 0.08:
            lines.append(b"")
        elif r < 0.16:
            lines.append(b"%d" % rng.choice([0, 1, -1]) + rng.choice([b"", b"\t", b" "]))
        else:
            toks = []
            for _ in range(rng.randrange(0, 8)):
                if rng.random() < 0.12:
                    toks.append(rng.choice(PIECES))
                else:
                    v = rng.choice([b"1", b"0.5", b"2", b"-3.25", b"0.001", b"%d.%d" % (rng.randrange(100), rng.randrange(1000))])
                    toks.append(b"%d:%d:%s" % (rng.randrange(40), rng.randrange(1000), v))
            sep = rng.choice([b" ", b"  ", b"\t"])
            lines.append(b"%d\t" % rng.choice([0, 1]) + sep.join(toks) + rng.choice([b"", b"", b"\r", b" "]))
    text = b"\n".join(lines)
    return text + (b"\n" if rng.random() < 0.7 else b"")


def test_seeded_fuzz_equals_the_host_loader(capi, tmp_path):
    rng = random.Random(2024)
    ctx = _dense(capi)
    for _ in range(300):
        text = _fuzz_doc(rng)
        try:
            ref = _reference(capi, text, tmp_path)
        except capi.LctrError:  # a stale %n can leave a wrapped id: the loader's error is raised on the device path too
            with pytest.raises(capi.LctrError, match="exceeds the device index types"):
                _upload(ctx, [text])
            continue
        for parts in _splits(text, rng, n_random=1)[::2]:
            got, _ = _upload(ctx, parts)
            _check_equal(got, ref)


# ---- 4. keyed contexts --------------------------------------------------------------------------------------------
def _keyed(capi, cap=4096, **kw):
    return capi.Context(capi.MODEL_FM, cap, 4, key_mode=capi.KEYS_HASHED, **kw)


KEYED_TEXT = (b"1\t0:%d:1 1:%d:0.5 2:77:2\n0\t\n1\t3:%d:1 4:77:1e-1 5:9\n0\t0:12345678901234567890:1\n"
              % (2 ** 32 + 5, 2 ** 40, 2 ** 63 + 1))


def test_keyed_insert_maps_rows_back_to_the_keys(capi, tmp_path):
    ref = _reference(capi, KEYED_TEXT, tmp_path, keyed=True)
    for parts in _splits(KEYED_TEXT, random.Random(3), n_random=1):
        ctx = _keyed(capi)
        (rp, rows, field, val, label), infos = _upload(ctx, parts)
        keys = ctx.download_keys()
        assert np.array_equal(keys[rows], ref.key)
        assert np.array_equal(rp, ref.row_ptr) and np.array_equal(field, ref.field)
        assert np.array_equal(val.view(np.uint32), ref.val.view(np.uint32))
        assert np.array_equal(label, ref.label[:ref.rows].astype(np.float32))
        assert sum(i.host_lines for i in infos) > 0  # the 20-digit id


def test_keyed_lookup_equals_upload_batch_keys(capi, tmp_path):
    ref = _reference(capi, KEYED_TEXT, tmp_path, keyed=True)
    ctx = _keyed(capi)
    ctx.upload_batch_keys(1, ref.row_ptr[:2], ref.key[:ref.row_ptr[1]], ref.field[:ref.row_ptr[1]], None, ref.label[:1])
    _upload(ctx, [KEYED_TEXT], slot=0, lookup=True)
    ctx.upload_batch_keys(1, ref.row_ptr, ref.key, ref.field, ref.val, ref.label[:ref.rows], insert=False)
    a, b = ctx.download_batch(0), ctx.download_batch(1)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    assert (a[1] == 4096).sum() > 0  # unseen keys sit on the null row (index = capacity)
    with pytest.raises(capi.LctrError, match="lookup only"):
        ctx.train_step(0)


def test_wide_ids_are_refused_on_dense_contexts(capi, tmp_path):
    p = str(tmp_path / "w.txt")
    open(p, "wb").write(KEYED_TEXT)
    with pytest.raises(capi.LctrError, match="exceed the device index types"):
        capi.load_libffm(p)
    with pytest.raises(capi.LctrError, match="line 1: .*exceeds the device index types"):
        _dense(capi).upload_libffm(0, KEYED_TEXT)


def test_keyed_admission_equals_upload_batch_keys(capi, tmp_path):
    rng = random.Random(5)
    text = b"".join(b"%d\t%s\n" % (rng.randrange(2), b" ".join(b"%d:%d:1" % (j, rng.randrange(60) * 7919 + 2 ** 33)
                                                              for j in range(rng.randrange(1, 9)))) for _ in range(200))
    ref = _reference(capi, text, tmp_path, keyed=True)
    a, b = _keyed(capi), _keyed(capi)
    for c in (a, b):
        c.set_key_admission(2, log2_width=12)
    # two uploads of the same text: the second admits the recurring keys
    for _ in range(2):
        a.upload_libffm(0, text)
        b.upload_batch_keys(0, ref.row_ptr, ref.key, ref.field, None, ref.label[:ref.rows])
        assert a.key_admission_stats() == b.key_admission_stats()
        (ra, fa, *xa), (rb, fb, *xb) = a.download_batch(0), b.download_batch(0)
        assert np.array_equal(ra, rb) and all(np.array_equal(x, y) for x, y in zip(xa, xb))
        # rows are handed out in arrival order on the device, which varies: compare the keys behind them
        assert np.array_equal(a.download_keys()[fa], b.download_keys()[fb])


# ---- 5. training from a text-uploaded slot ------------------------------------------------------------------------
def _train_text(rng, F, fields, ones):
    lines = []
    for _ in range(256):
        toks = [b"%d:%d:%s" % (f, rng.randrange(F), b"1" if ones else rng.choice([b"1", b"0.5", b"2.25", b"0.125"]))
                for f in range(fields) if rng.random() < 0.8]
        lines.append(b"%d\t%s" % (rng.randrange(2), b" ".join(toks)))
    return b"\n".join(lines) + b"\n"


TRAIN_CASES = {
    "fm_k16_det0": dict(model=1, k=16, kw={}),
    "fm_k16_det2": dict(model=1, k=16, kw=dict(deterministic=2)),
    "ffm_k4": dict(model=2, k=4, kw={}),
    "nfm_bf16": dict(model=3, k=16, kw=dict(hidden=(32, 16), mlp_precision=1)),
    "wnd": dict(model=4, k=4, kw=dict(hidden=(32,))),
}


@pytest.mark.parametrize("ones", [True, False], ids=["val_absent", "val_present"])
@pytest.mark.parametrize("case", sorted(TRAIN_CASES))
def test_training_from_text_equals_host_csr(capi, tmp_path, case, ones):
    c = TRAIN_CASES[case]
    F, Fc = 500, 8
    text = _train_text(random.Random(11), F, Fc, ones)
    ref = _reference(capi, text, tmp_path)
    runs = []
    for use_text in (True, False):
        ctx = capi.Context(c["model"], F, c["k"], field_cnt=Fc, minibatch_size=ref.rows, **c["kw"])
        ctx.fill_params(7, 0.05)
        if use_text:
            info = ctx.upload_libffm(0, text)
            assert info.host_lines == 0 and info.rows == ref.rows
        else:
            ctx.upload_dataset(0, ref)
        losses = [ctx.train_step(0) for _ in range(3)]
        runs.append((losses, ctx.download_params()))
    (la, (Wa, Va)), (lb, (Wb, Vb)) = runs
    if case == "fm_k16_det2":  # the grouped backward is order-fixed: bit for bit
        assert la == lb and np.array_equal(Wa, Wb) and np.array_equal(Va, Vb)
    else:  # the other paths sum gradients with atomics, whose order varies from run to run
        np.testing.assert_allclose(la, lb, rtol=1e-5)
        np.testing.assert_allclose(Wa, Wb, rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(Va, Vb, rtol=1e-4, atol=1e-6)


# ---- 6. refusals and failures -------------------------------------------------------------------------------------
def test_refusals(capi):
    with pytest.raises(capi.LctrError, match="deterministic = 1"):
        _dense(capi, deterministic=1).upload_libffm(0, b"1\t0:1:1\n")
    with pytest.raises(capi.LctrError, match="out of range"):
        _dense(capi).upload_libffm(8, b"1\t0:1:1\n")
    with pytest.raises(capi.LctrError, match="LCTR_TEXT_LOOKUP needs a keyed context"):
        _dense(capi).upload_libffm(0, b"1\t0:1:1\n", lookup=True)
    two = capi.Context(capi.MODEL_FM, 1000, 16, world=2, rank=0, minibatch_size=64)
    with pytest.raises(capi.LctrError, match="single-GPU"):
        two.upload_libffm(0, b"1\t0:1:1\n")


def test_upload_errors_name_the_line(capi):
    with pytest.raises(capi.LctrError, match="line 3: a fid >= feature_cnt 1000"):
        _dense(capi).upload_libffm(0, b"1\t0:1:1\n0\t\n1\t0:1000:1\n")
    with pytest.raises(capi.LctrError, match="line 2: a fid >= feature_cnt 1000"):  # a line the host parses
        _dense(capi).upload_libffm(0, b"1\t0:1:1\n0\t0:5000:1e0\n")
    ffm = capi.Context(capi.MODEL_FFM, 1000, 4, field_cnt=4)
    with pytest.raises(capi.LctrError, match="line 2: a field >= field_cnt 4"):
        ffm.upload_libffm(0, b"1\t0:1:1\n0\t4:2:1\n")
    with pytest.raises(capi.LctrError, match="line 4: a fid / field exceeds"):  # counted across calls
        ffm.upload_libffm(0, b"1\t0:1:1\n0\t1:2:1\n", end=False)
        ffm.upload_libffm(0, b"1\t0:1:1\n0\t70000:2:1\n", begin=False)


def test_a_failed_call_changes_no_state_and_leaves_the_slot_unusable(capi, tmp_path):
    good = [b"1\t0:3:2.5\n1\t\n", b"0\t1:4 2:5:1\n1\t0:1:1\n"]
    ref = _reference(capi, b"".join(good), tmp_path)
    ctx = _dense(capi)
    ctx.upload_libffm(0, good[0], end=False)
    first = ctx.download_batch(0)
    with pytest.raises(capi.LctrError, match="feature_cnt"):
        ctx.upload_libffm(0, b"0\t0:7:9 1:99999:1\n", begin=False, end=False)
    with pytest.raises(capi.LctrError, match="no usable batch"):
        ctx.train_step(0)
    ctx.upload_libffm(0, good[1], begin=False, end=True)  # continues from the state before the failed call
    second = ctx.download_batch(0)
    rp = np.concatenate([first[0], second[0][1:] + first[0][-1]])
    got = [rp] + [np.concatenate([a, b]) for a, b in zip(first[1:], second[1:])]
    _check_equal(got, ref)
    ctx.train_step(0)
