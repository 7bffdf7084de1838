"""tests/ref64.py against the CPU oracle (and against its own derivatives), so that the GPU shape tests can lean on it.

The oracle computes in fp32 in the reference's order; ref64 in float64 from the definitions.  They must agree within
fp32 rounding of the sums involved: |oracle - ref64| <= 1e-5 * cond + 1e-7, cond being ref64's absolute-value figure."""
import numpy as np
import pytest

import ref64


def _batch(rng, F, rows, Fc=0, with_val=True):
    lens = rng.integers(2, 30, rows)
    lens[:5] = (0, 1, 63, 64, 65)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fid = np.concatenate([rng.choice(F, n, replace=False) for n in lens]).astype(np.uint32)
    fld = rng.integers(0, max(Fc, 1), len(fid)).astype(np.uint32)
    val = (0.5 + rng.random(len(fid))).astype(np.float32) if with_val else np.ones(len(fid), np.float32)
    lab = (rng.random(rows) < 0.4).astype(np.int32)
    return rp, fid, fld, val, lab


def _close(got, want, cond, rtol=1e-5, atol=1e-7):
    err = np.abs(np.asarray(got, np.float64) - want)
    bound = rtol * cond + atol
    return bool(np.all(err <= bound)), float(np.max(err - bound))


@pytest.mark.parametrize("k,with_val", [(3, True), (8, False), (24, True)])
def test_fm_forward_and_gradient_match_the_oracle(oracle_api, k, with_val):
    rng = np.random.default_rng(k)
    F, rows = 300, 40
    rp, fid, fld, val, lab = _batch(rng, F, rows, with_val=with_val)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    V = (rng.standard_normal(F * k) * 0.3 / np.sqrt(k)).astype(np.float32)
    ds = oracle_api.Dataset(rp, fid, fld, val, lab, F, 0)
    o = oracle_api.FMOracle(ds, k, W, V)
    o.forward_backward()
    s64, z64, p64, s_c, z_c = ref64.fm_forward(rp, fid, val, W, V, k)
    ok, ex = _close(o.sumVX.reshape(rows, k), s64, s_c)
    assert ok, ex
    # pCTR: the logit bound carried through the sigmoid's slope, plus the fp32 sigmoid's own rounding
    ok, ex = _close(o.pred, p64, p64 * (1 - p64) * z_c, atol=3e-7)
    assert ok, ex
    gW, gV, gW_c, gV_c = ref64.fm_grad(rp, fid, val, lab, W, V, k, o.pred, o.sumVX, float(o.l2))
    ok, ex = _close(o.update_g[:F], gW, gW_c)
    assert ok, ex
    ok, ex = _close(o.update_g[F:].reshape(F, k), gV, gV_c)
    assert ok, ex
    assert np.count_nonzero(gV) > F  # the batch touches most features


@pytest.mark.parametrize("Fc,k,with_val", [(5, 2, True), (7, 3, False), (13, 1, True)])
def test_ffm_forward_gradient_and_predict_match_the_oracle(oracle_api, Fc, k, with_val):
    rng = np.random.default_rng(Fc * 10 + k)
    F, rows = 200, 30
    rp, fid, fld, val, lab = _batch(rng, F, rows, Fc, with_val)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    V = (rng.standard_normal(F * Fc * k) * 0.1).astype(np.float32)
    ds = oracle_api.Dataset(rp, fid, fld, val, lab, F, Fc)
    o = oracle_api.FFMOracle(ds, k, W, V)
    o.forward_backward()
    z64, p64, z_c = ref64.ffm_forward(rp, fid, fld, val, W, V, Fc, k)
    ok, ex = _close(o.pred, p64, p64 * (1 - p64) * z_c, atol=3e-7)
    assert ok, ex
    gW, gV, gW_c, gV_c = ref64.ffm_grad(rp, fid, fld, val, lab, W, V, Fc, k, o.pred, float(o.l2))
    ok, ex = _close(o.update_g[:F], gW, gW_c)
    assert ok, ex
    ok, ex = _close(o.update_g[F:].reshape(F, Fc, k), gV, gV_c)
    assert ok, ex
    pctr, _, _, _ = oracle_api.predict(ds, Fc, k, W, V, None, True)
    ok, ex = _close(pctr, p64, p64 * (1 - p64) * z_c, atol=3e-7)
    assert ok, ex


def test_nfm_sumvx_matches_the_oracle(oracle_api):
    rng = np.random.default_rng(4)
    F, rows, k = 300, 40, 6
    rp, fid, fld, val, lab = _batch(rng, F, rows)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    V = (rng.standard_normal(F * k) * 0.2).astype(np.float32)
    ds = oracle_api.Dataset(rp, fid, fld, val, lab, F, 0)
    o = oracle_api.NFMOracle(ds, k, [8], W=W, V=V, batch_size=rows, minibatch=rows)
    o.epoch()  # one minibatch: sumVX is formed from the initial V
    _z, _wide, s64, _zc, _wc = ref64.nfm_forward(rp, fid, val, W, V, k)
    s_c = ref64.fm_forward(rp, fid, val, W, V, k)[3]
    ok, ex = _close(o.sumVX.reshape(rows, k), s64, s_c)
    assert ok, ex


def _num_grad(fun, a, idx, h=1e-6):
    out = []
    for i in idx:
        ap, am = a.copy(), a.copy()
        ap[i] += h
        am[i] -= h
        out.append((fun(ap) - fun(am)) / (2 * h))
    return np.array(out)


def test_fm_and_nfm_gradients_are_the_derivatives():
    """With l2 = 0, fm_grad is d/dV of sum_r (p_r - y_r) logit_r(V) at fixed p, and nfm_grad is d/dV of
    sum_r <dz_r, z_r(V)>: central differences in float64 agree to 1e-6 relative."""
    rng = np.random.default_rng(6)
    F, rows, k = 100, 12, 5
    rp, fid, _fld, val, lab = _batch(rng, F, rows)
    val = val.astype(np.float64)
    W = rng.standard_normal(F) * 0.1
    V = rng.standard_normal(F * k) * 0.3
    p = rng.random(rows)
    dz = rng.standard_normal((rows, k))
    d = p - lab
    s = ref64.fm_forward(rp, fid, val, W, V, k)[0]
    gW, gV, _, _ = ref64.fm_grad(rp, fid, val, lab, W, V, k, p, s, 0.0)
    hot = np.unique(fid)[:6]
    idxV = (hot[:, None] * k + np.arange(k)).ravel()
    numV = _num_grad(lambda v: np.dot(d, ref64.fm_forward(rp, fid, val, W, v, k)[1]), V, idxV)
    numW = _num_grad(lambda w: np.dot(d, ref64.fm_forward(rp, fid, val, w, V, k)[1]), W, hot)
    assert np.allclose(gV.ravel()[idxV], numV, rtol=1e-6, atol=1e-8)
    assert np.allclose(gW[hot], numW, rtol=1e-6, atol=1e-8)
    _, gVn, _, _ = ref64.nfm_grad(rp, fid, val, lab, W, V, k, p, s, dz, 0.0)
    numVn = _num_grad(lambda v: np.sum(dz * ref64.nfm_forward(rp, fid, val, W, v, k)[0]), V, idxV)
    assert np.allclose(gVn.ravel()[idxV], numVn, rtol=1e-6, atol=1e-8)


def test_ffm_gradient_skips_rows_whose_prediction_equals_the_label():
    rng = np.random.default_rng(8)
    F, rows, Fc, k = 100, 10, 4, 2
    rp, fid, fld, val, lab = _batch(rng, F, rows, Fc)
    W = rng.standard_normal(F) * 0.1
    V = rng.standard_normal(F * Fc * k) * 0.3
    p = rng.random(rows)
    p[3], p[7] = lab[3], lab[7]
    got = ref64.ffm_grad(rp, fid, fld, val, lab, W, V, Fc, k, p, 0.001)
    keep = np.array([r for r in range(rows) if r not in (3, 7)])
    lens = np.diff(rp)[keep]
    sel = np.concatenate([np.arange(rp[r], rp[r + 1]) for r in keep])
    rp2 = np.concatenate([[0], np.cumsum(lens)])
    want = ref64.ffm_grad(rp2, fid[sel], fld[sel], val[sel], lab[keep], W, V, Fc, k, p[keep], 0.001)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
