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


def _adagrad_recovered(w0, w1, accum, B):
    """the gradient behind one oracle Adagrad step from a zero state: |g| = sqrt(accum) * B (accum = (g / B)^2), the sign
    from the step; returns (g, sign_known)"""
    mag = np.sqrt(accum.astype(np.float64)) * B
    step = w0.astype(np.float64) - w1.astype(np.float64)
    return np.sign(step) * mag, step != 0


@pytest.mark.parametrize("act,hidden", [(0, [8]), (1, [8]), (0, [7, 5])], ids=["sigmoid-H8", "tanh-H8", "sigmoid-H7-5"])
def test_nfm_head_and_gradient_match_the_oracle(oracle_api, act, hidden):
    """One minibatch of NFMOracle from a zero Adagrad state (masks all 1, biases != 0): the loss from nfm_head's pCTR, and
    the gradient recovered from the step (|g| from the accumulator, the sign from the step) against nfm_head + nfm_grad,
    within 1e-5 of their condition figures (the oracle's own fp32 dz folded into gV's)."""
    rng = np.random.default_rng(20 + act + len(hidden))
    F, rows, k = 300, 40, 6
    rp, fid, fld, val, lab = _batch(rng, F, rows)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    V = (rng.standard_normal(F * k) * 0.3).astype(np.float32)
    ds = oracle_api.Dataset(rp, fid, fld, val, lab, F, 0)
    o = oracle_api.NFMOracle(ds, k, hidden, W=W, V=V, batch_size=rows, minibatch=rows, lr=1.0, act=act)
    layers = []
    for l in range(len(hidden) + 1):
        o.mlp.arrays("mask", l)[:] = 1.0
        o.mlp.arrays("bias", l)[:] = (rng.standard_normal(len(o.mlp.arrays("bias", l))) * 0.1).astype(np.float32)
        layers.append((o.mlp.arrays("weight", l).copy(), o.mlp.arrays("bias", l).copy()))
    loss, _ = o.epoch()
    z, wide, s64, z_c, w_c = ref64.nfm_forward(rp, fid, val, W, V, k)
    p, dz, dz_c, _lc = ref64.nfm_head(z, wide, layers, act, None, lab, z_c, w_c)
    loss64 = float(np.sum(np.where(lab == 1, -np.log(p), -np.log(1 - p))))
    assert abs(loss - loss64) <= 1e-5 * loss64, (loss, loss64)
    gW, gV, gW_c, gV_c = ref64.nfm_grad(rp, fid, val, lab, W, V, k, p, s64, dz, float(o.l2), dz_cond=dz_c)
    for w0, w1, acc, g, c in ((W, o.W, o.accum[:F], gW, gW_c), (V, o.V, o.accum[F:], gV.ravel(), gV_c.ravel())):
        got, known = _adagrad_recovered(w0, w1, acc, rows)
        err = np.where(known, np.abs(got - g), np.minimum(np.abs(got - g), np.abs(-got - g)))
        bound = 1e-5 * c + 1e-7
        assert np.all(err <= bound), float(np.max(err - bound))
    assert np.count_nonzero(gV) > F  # the batch touches most features


def _wnd_batch(rng, F, rows, Fc, with_val=True):
    """_batch's rows (0, 1, 63, 64 and 65 entries first, fields unsorted and repeated, fields absent), plus: in the
    63-entry row a fid repeated and one fid that is the first entry of two fields; in the 64-entry row a field whose
    entries all lie past the 32nd"""
    rp, fid, fld, val, lab = _batch(rng, F, rows, Fc, with_val)
    b = rp[2]
    fid[b + 40] = fid[b + 3]                                         # the same fid twice in a row
    fld[b:b + 63][fld[b:b + 63] == (fld[b] + 1) % Fc] = (fld[b] + 2) % Fc
    fid[b + 1], fld[b + 1] = fid[b], (fld[b] + 1) % Fc               # fid of entry 0 first of a second field
    b = rp[3]
    late = (fld[b] + 1) % Fc
    fld[b:b + 32][fld[b:b + 32] == late] = fld[b]
    fld[b + 50] = late                                               # field `late` only past entry 31
    return rp, fid, fld, val, lab


def _wnd_layers(rng, dims):
    return [((rng.random((dims[i + 1], dims[i])) - 0.5).astype(np.float32) * np.float32(2 / np.sqrt(dims[i])),
             (rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32)) for i in range(len(dims) - 1)]


@pytest.mark.parametrize("Fc,d,act,hidden,with_val", [(13, 4, 0, [8], True), (6, 3, 1, [8], False),
                                                      (40, 2, 0, [7, 5], True)],
                         ids=["Fc13-d4-sigmoid-H8", "Fc6-d3-tanh-H8", "Fc40-d2-sigmoid-H7-5"])
def test_wnd_forward_gradient_and_dense_gradients_match_the_oracle(oracle_api, Fc, d, act, hidden, with_val):
    """One minibatch of WNDOracle with the parameter-server SGD rule and lr = minibatch, so that g = w0 - w1 for W and E
    (ref64.probe_excess), and its dense layers from a zero Adagrad state (masks all 1) recovered as in the NFM test; the
    loss from nfm_head's pCTR on wnd_forward's z."""
    rng = np.random.default_rng(40 + Fc + d)
    F, rows = 300, 40
    rp, fid, fld, val, lab = _wnd_batch(rng, F, rows, Fc, with_val)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    E = (rng.standard_normal(F * d) * 0.3).astype(np.float32)
    ds = oracle_api.Dataset(rp, fid, fld, val, lab, F, Fc)
    o = oracle_api.WNDOracle(ds, d, hidden, W, E, lr=float(rows), batch_size=rows, minibatch=rows, act=act,
                             optimizer="ps_sgd")
    dims = [Fc * d] + hidden + [1]
    layers = _wnd_layers(rng, dims)
    for l, (w, b) in enumerate(layers):
        o.mlp.arrays("mask", l)[:] = 1.0
        o.mlp.arrays("weight", l)[:] = w.ravel()
        o.mlp.arrays("bias", l)[:] = b
    loss, _ = o.epoch()
    z, first, wide, z_c, w_c = ref64.wnd_forward(rp, fid, fld, val, W, E, Fc, d)
    assert np.sum(first[2] == fid[rp[2]]) == 2                       # one fid first of two fields
    p, dz, dz_c, _lc, dense = ref64.nfm_head(z, wide, layers, act, None, lab, z_c, w_c, grads=True)
    loss64 = float(np.sum(np.where(lab == 1, -np.log(p), -np.log(1 - p))))
    assert abs(loss - loss64) <= 1e-5 * loss64, (loss, loss64)
    gW, gE, gW_c, gE_c = ref64.wnd_grad(rp, fid, fld, val, lab, W, E, Fc, d, p, dz, float(o.l2), dz_cond=dz_c)
    for name, w0, w1, g, c in (("W", W, o.W, gW, gW_c), ("E", E, o.E, gE.ravel(), gE_c.ravel())):
        ex = ref64.probe_excess(w0.astype(np.float64) - w1, g, c, w1)
        assert np.all(ex <= 0), (name, float(np.max(ex)), int(np.argmax(ex)))
    moved = np.flatnonzero(np.any(o.E.reshape(F, d) != E.reshape(F, d), 1))
    assert np.array_equal(moved, np.unique(first[first >= 0]))      # only first-of-field tensors move
    for l in range(len(dims) - 1):
        acc = o.mlp.arrays("accum", l)
        out = dims[l + 1]
        dW, db, dW_c, db_c = dense[l]
        for w0, w1, a, g, c in ((layers[l][1], o.mlp.arrays("bias", l), acc[:out], db, db_c),
                                (layers[l][0].ravel(), o.mlp.arrays("weight", l), acc[out:], dW.ravel(), dW_c.ravel())):
            got, known = _adagrad_recovered(w0, w1, a, rows)
            err = np.where(known, np.abs(got - g), np.minimum(np.abs(got - g), np.abs(-got - g)))
            bound = 1e-5 * c + 1e-7
            assert np.all(err <= bound), (l, float(np.max(err - bound)))


def test_wnd_gradients_are_the_derivatives():
    """With l2 = 0, for the weighted loss L = sum_r w_r logloss(p_r) of the whole float64 Wide&Deep model (wnd_forward +
    nfm_head, no delta reaching the +-15 clip): wnd_grad's gW and gE and nfm_head's dense gradients agree with central
    differences of L to 1e-6 relative, on rows with repeated fields and fids."""
    rng = np.random.default_rng(12)
    F, rows, Fc, d = 100, 10, 5, 3
    rp, fid, fld, val, lab = _wnd_batch(rng, F, rows, Fc)
    val = val.astype(np.float64)
    W = rng.standard_normal(F) * 0.1
    E = rng.standard_normal(F * d) * 0.3
    layers = [(w.astype(np.float64), b.astype(np.float64)) for w, b in _wnd_layers(rng, [Fc * d, 6, 4, 1])]
    rw = 0.25 + 2 * rng.random(rows)

    def loss(W_, E_, layers_):
        z, _f, wide, _zc, _wc = ref64.wnd_forward(rp, fid, fld, val, W_, E_, Fc, d)
        p = ref64.nfm_head(z, wide, layers_, 1, None, lab)[0]
        return float(np.sum(rw * np.where(lab == 1, -np.log(p), -np.log(1 - p))))

    z, first, wide, _zc, _wc = ref64.wnd_forward(rp, fid, fld, val, W, E, Fc, d)
    p, dz, _dc, _lc, dense = ref64.nfm_head(z, wide, layers, 1, None, lab, weights=rw, grads=True)
    gW, gE, _, _ = ref64.wnd_grad(rp, fid, fld, val, lab, W, E, Fc, d, p, dz, 0.0, weights=rw)
    firsts = np.unique(first[first >= 0])
    seen_late = np.setdiff1d(np.unique(fid), firsts)                 # fids never first of a field: gE = 0
    assert len(seen_late) > 0 and np.all(gE[seen_late] == 0)
    idxE = (firsts[:8, None] * d + np.arange(d)).ravel()
    numE = _num_grad(lambda e: loss(W, e, layers), E, idxE)
    assert np.allclose(gE.ravel()[idxE], numE, rtol=1e-6, atol=1e-8)
    ids = np.unique(fid)[:8]
    assert np.allclose(gW[ids], _num_grad(lambda w: loss(w, E, layers), W, ids), rtol=1e-6, atol=1e-8)
    for l in range(len(layers)):
        def with_layer(wb, l=l, part=0):
            out = list(layers)
            out[l] = (wb.reshape(layers[l][0].shape), layers[l][1]) if part == 0 else (layers[l][0], wb)
            return out
        w, b = layers[l]
        iw = np.arange(0, w.size, max(1, w.size // 7))
        numw = _num_grad(lambda v: loss(W, E, with_layer(v)), w.ravel(), iw)
        assert np.allclose(dense[l][0].ravel()[iw], numw, rtol=1e-6, atol=1e-8), l
        numb = _num_grad(lambda v: loss(W, E, with_layer(v, part=1)), b, np.arange(len(b)))
        assert np.allclose(dense[l][1], numb, rtol=1e-6, atol=1e-8), l


def _hot_fm_problem(rows=2000, F=500, k=8, seed=31):
    """every row holds id 0; returns the batch, parameters, the float64 forward and gradient"""
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 20, rows)
    fid = np.concatenate([np.concatenate([[0], rng.choice(np.arange(1, F), n - 1, replace=False)]) for n in lens])
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    val = (0.25 + 1.5 * rng.random(len(fid))).astype(np.float32)
    lab = (rng.random(rows) < 0.4).astype(np.int32)
    W = (rng.standard_normal(F) * 0.05).astype(np.float32)
    V = (rng.standard_normal(F * k) * 0.1 / np.sqrt(k)).astype(np.float32)
    return rp, fid.astype(np.uint32), val, lab, W, V


def test_probe_bound_sees_a_dropped_or_doubled_share():
    """The bound of the gradient probe (ref64.probe_excess) on the feature with the most rows: leaving out its largest
    single-row term, or counting one of 32 replica shares twice, leaves the bound on every coordinate; so does an NFM dz
    read from the neighbouring sample, and an FFM l2 count c_ib one too high at l2 = 5e-2 (on every touched row, and on
    all but the factors whose V is near 0)."""
    k, l2 = 8, 0.001
    rp, fid, val, lab, W, V = _hot_fm_problem(k=k)
    rows = len(lab)
    s, _z, p, _sc, _zc = ref64.fm_forward(rp, fid, val, W, V, k)
    gW, gV, gW_c, gV_c = ref64.fm_grad(rp, fid, val, lab, W, V, k, p, s, l2)
    at = np.flatnonzero(fid == 0)
    r = np.repeat(np.arange(rows), np.diff(rp))[at]
    x = val[at].astype(np.float64)
    gw_r = (p[r] - lab[r]) * x + l2 * W[0]
    gv_r = (s[r] - x[:, None] * V[:k].astype(np.float64)) * gw_r[:, None] + l2 * V[:k]
    terms = np.concatenate([gw_r[:, None], gv_r], 1)                      # [rows of id 0, 1 + k]
    g = np.concatenate([[gW[0]], gV[0]])
    cond = np.concatenate([[gW_c[0]], gV_c[0]])
    w1 = (np.concatenate([[W[0]], V[:k]]).astype(np.float64) - g).astype(np.float32)
    dropped = g - terms[np.argmax(np.abs(terms), 0), np.arange(k + 1)]
    assert np.all(ref64.probe_excess(dropped, g, cond, w1) > 0)
    doubled = g + terms[r % 32 == 5].sum(0)
    assert np.all(ref64.probe_excess(doubled, g, cond, w1) > 0)
    # NFM: dz of the neighbouring sample
    rng = np.random.default_rng(3)
    layers = [(rng.random((16, k)) - 0.5, np.zeros(16)), (rng.random((1, 16)) - 0.5, np.zeros(1))]
    z, wide, s64, z_c, w_c = ref64.nfm_forward(rp, fid, val, W, V, k)
    pn, dz, dz_c, _ = ref64.nfm_head(z, wide, layers, 0, None, lab, z_c, w_c)
    _, gVn, _, gVn_c = ref64.nfm_grad(rp, fid, val, lab, W, V, k, pn, s64, dz, l2, dz_cond=dz_c)
    _, gVs, _, _ = ref64.nfm_grad(rp, fid, val, lab, W, V, k, pn, s64, np.roll(dz, 1, 0), l2)
    w1n = (V[:k].astype(np.float64) - gVn[0]).astype(np.float32)
    assert np.all(ref64.probe_excess(gVs[0], gVn[0], gVn_c[0], w1n) > 0)
    # FFM: c_ib = cnt[b] instead of cnt[b] - 1 for the entry's own field b = a_i
    Fc, kf, l2f = 6, 4, 5e-2
    rp2, fid2, fld2, val2, lab2 = _batch(np.random.default_rng(9), 200, 30, Fc)
    Wf = (rng.standard_normal(200) * 0.05).astype(np.float32)
    Vf = (rng.standard_normal(200 * Fc * kf) * 0.1).astype(np.float32)
    _z, pf, _c = ref64.ffm_forward(rp2, fid2, fld2, val2, Wf, Vf, Fc, kf)
    _, gVf, _, gVf_c = ref64.ffm_grad(rp2, fid2, fld2, val2, lab2, Wf, Vf, Fc, kf, pf, l2f)
    V3 = Vf.reshape(-1, Fc, kf).astype(np.float64)
    bad = gVf.copy()
    hit = np.zeros(gVf.shape[:2], bool)
    for row in range(len(lab2)):
        f, a = fid2[rp2[row]:rp2[row + 1]].astype(np.int64), fld2[rp2[row]:rp2[row + 1]].astype(np.int64)
        cnt = np.bincount(a, minlength=Fc)
        for fi, ai in zip(f, a):
            if cnt[ai] > 1:
                bad[fi, ai] += l2f * V3[fi, ai]
                hit[fi, ai] = True
    w1f = (V3 - gVf).astype(np.float32)
    assert hit.sum() > 10
    out = ref64.probe_excess(bad, gVf, gVf_c, w1f)[hit]
    assert np.mean(out > 0) > 0.95 and np.all(out.max(1) > 0)  # only factors with V ~ 0 may stay inside
