"""Weighted test-set metrics on the GPU (lctr_eval_pred_weighted, lctr_eval_weighted) against the numpy restatement of
their rule (tests/weighted_eval.py): AUC and the weighted correct count bit for bit, the logloss within 1e-6 relative
(the device's logf / log against numpy's)."""
import numpy as np
import pytest

import weighted_eval as we

pytestmark = pytest.mark.gpu

F = 2000


@pytest.fixture(scope="module")
def ctx():
    from lightctr_b200 import capi
    c = capi.Context(capi.MODEL_FM, F, 8)
    yield c
    c.close()


def _bits(x):
    return np.float32(x).view(np.uint32)


def _same(got, want, loss=True):
    assert _bits(got[2]) == _bits(want[2]), ("auc", got[2], want[2])
    assert got[1] == want[1], ("correct", got[1], want[1])
    if loss:
        np.testing.assert_allclose(got[0], want[0], rtol=1e-6)


def _rows(n, seed):
    rng = np.random.default_rng(seed)
    return rng.random(n).astype(np.float32), (rng.random(n) < 0.25).astype(np.int32), rng


CASES = ["random_1m", "ties", "all_positive", "huge", "tiny"]


def _case(name):
    if name == "random_1m":
        p, y, rng = _rows(1 << 20, 1)
        w = (rng.random(len(p)) * 5).astype(np.float32)
        w[rng.random(len(p)) < 0.1] = 0.0
    elif name == "ties":  # p saturated at 0 and 1 on most rows
        p, y, rng = _rows(200000, 2)
        p = np.where(rng.random(len(p)) < 0.8, (rng.random(len(p)) < 0.5).astype(np.float32), p).astype(np.float32)
        w = rng.integers(0, 4, len(p)).astype(np.float32) * np.float32(0.75)
    elif name == "all_positive":
        p, y, rng = _rows(50000, 3)
        y[:] = 1
        w = (rng.random(len(p)) * 2).astype(np.float32)
    elif name == "huge":
        p, y, rng = _rows(100000, 4)
        w = (3e38 * (0.5 + 0.5 * rng.random(len(p)))).astype(np.float32)
        w[::3] = (rng.random(len(w[::3])) * 1e30).astype(np.float32)
    else:
        p, y, rng = _rows(100000, 5)
        w = (1e-30 * (0.5 + rng.random(len(p)))).astype(np.float32)
    return p, y, w


@pytest.mark.parametrize("name", CASES)
def test_matches_the_rule(ctx, name):
    p, y, w = _case(name)
    with np.errstate(over="ignore"):
        want = we.eval_weighted(p, y, w)
    _same(ctx.eval_pred(p, y, w), want)


def test_unit_weights_equal_eval_pred(ctx):
    p, y, _ = _rows(300000, 6)
    p[:1000] = 0.0
    p[1000:2000] = 1.0
    a = ctx.eval_pred(p, y, np.ones(len(p), np.float32))
    b = ctx.eval_pred(p, y)
    assert _bits(a[0]) == _bits(b[0]) and a[1] == float(b[1]) and _bits(a[2]) == _bits(b[2]), (a, b)


def test_integer_weights_equal_expanded_rows(ctx):
    p, y, rng = _rows(200000, 7)
    w = rng.integers(0, 5, len(p))
    a = ctx.eval_pred(p, y, w.astype(np.float32))
    rows = np.repeat(np.arange(len(p)), w)
    b = ctx.eval_pred(p[rows], y[rows])
    assert a[1] == float(b[1]) and _bits(a[2]) == _bits(b[2]), (a, b)


def test_zero_weights_equal_filtered_rows(ctx):
    p, y, rng = _rows(200000, 8)
    w = (rng.random(len(p)) * 3).astype(np.float32)
    w[rng.random(len(p)) < 0.3] = 0.0
    p[::97] = 1.0  # -log(1 - p) = inf on a negative row: a zero weight must not turn it into 0 * inf
    y[::97] = 0
    w[::97] = 0.0
    keep = w != 0
    a = ctx.eval_pred(p, y, w)
    b = ctx.eval_pred(p[keep], y[keep], w[keep])
    assert _bits(a[0]) == _bits(b[0]) and a[1] == b[1] and _bits(a[2]) == _bits(b[2]), (a, b)
    assert np.isfinite(a[0])


def test_shuffle_and_repeat_keep_the_auc(ctx):
    p, y, rng = _rows(500000, 9)
    w = (rng.random(len(p)) * 7).astype(np.float32)
    a = ctx.eval_pred(p, y, w)
    assert ctx.eval_pred(p, y, w) == a
    perm = rng.permutation(len(p))
    assert _bits(ctx.eval_pred(p[perm], y[perm], w[perm])[2]) == _bits(a[2])


def test_unweighted_calls_keep_their_bits_in_between(ctx):
    from lightctr_b200.data import CriteoSynth
    rp, fid, _fld, lab = CriteoSynth(F, seed=3).batch(4096)
    ctx.upload_batch(1, rp, fid, None, None, lab)
    ctx.predict(1)
    p, y, rng = _rows(100000, 10)
    e0, u0 = ctx.eval_metrics(1), ctx.eval_pred(p, y)
    for i in range(3):
        ctx.eval_pred(p, y, (rng.random(len(p)) * (i + 1)).astype(np.float32))
        assert ctx.eval_metrics(1) == e0
        assert ctx.eval_pred(p, y) == u0


def test_slot_weights_equal_host_arrays_and_refusals(ctx):
    from lightctr_b200 import capi
    from lightctr_b200.data import CriteoSynth
    rp, fid, _fld, lab = CriteoSynth(F, seed=4).batch(8192)
    ctx.upload_batch(2, rp, fid, None, None, lab)
    with pytest.raises(capi.LctrError, match="no row weights"):
        ctx.eval_weighted(2)
    w = (np.random.default_rng(11).random(len(lab)) * 3).astype(np.float32)
    w[::5] = 0.0
    ctx.set_row_weights(2, w)
    pctr = ctx.score(2)
    _same(ctx.eval_weighted(2), ctx.eval_pred(pctr, lab, w))
    _same(ctx.eval_weighted(2), we.eval_weighted(pctr, lab, w))
    n = ctx.launch_count()
    for bad in (np.nan, -1.0, np.inf):
        wb = w.copy()
        wb[17] = bad
        with pytest.raises(capi.LctrError, match="not a finite value"):
            ctx.eval_pred(pctr, lab, wb)
    assert ctx.launch_count() == n  # a refused call launches nothing
    ctx.upload_batch(2, rp, fid, None, None, lab)  # an upload drops the weights
    with pytest.raises(capi.LctrError, match="no row weights"):
        ctx.eval_weighted(2)
