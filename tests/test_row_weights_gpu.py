"""Per-row weights (lctr_set_row_weights) on the GPU.

The float64 oracle of a weighted step is g64 = sum_r w_r g64(row r alone), each row's gradient from tests/ref64.py; the
GPU gradient comes from one unit SGD step (OPT_PS_SGD, lr = minibatch_size = 1, so g = w0 - w1) and is held to
|g - g64| <= 1e-5 cond + spacing(w1) with cond = sum_r w_r cond_r.  NFM's weighted head (clip on w (p - y)) is built
from ref64.nfm_head's pieces here."""
import os
import subprocess
import sys

import numpy as np
import pytest

import ref64
from kernel_shapes_worker import make_batch, make_params

pytestmark = pytest.mark.gpu

L2 = 0.001
NFM_H = 16


def _weights(rows, seed, zeros=True):
    rng = np.random.default_rng(seed)
    w = (rng.random(rows) * 4).astype(np.float32)
    if zeros:
        w[rng.choice(rows, max(1, rows // 10), replace=False)] = 0.0
    return w


def _row(batch, r):
    rp, fid, fld, val, lab = batch
    b, e = rp[r], rp[r + 1]
    return np.array([0, e - b], np.int64), fid[b:e], fld[b:e], None if val is None else val[b:e], lab[r:r + 1]


def _ctx(model, F, k, Fc=0, **kw):
    from lightctr_b200 import capi
    return capi.Context(model, F, k, Fc, optimizer=capi.OPT_PS_SGD, lr=1.0, minibatch_size=1, l2=L2, **kw)


def _upload(ctx, slot, batch, Fc=0):
    rp, fid, fld, val, lab = batch
    ctx.upload_batch(slot, rp, fid, fld if Fc else None, val, lab)


def _check_grad(what, w0, w1, g64, cond, rtol=1e-5):
    got = w0.astype(np.float64) - w1.astype(np.float64)
    ex = ref64.probe_excess(got, g64.ravel(), cond.ravel(), w1, rtol)
    at = int(np.argmax(ex))
    assert ex[at] <= 0, (what, float(ex[at]), at, float(got[at]), float(g64.ravel()[at]), float(cond.ravel()[at]))


def fm_weighted64(batch, W0, V0, k, pred, w, l2=L2):
    """sum_r w_r * ref64.fm_grad(row r alone), with the step's own pCTR"""
    rp, fid, fld, val, lab = batch
    s64 = ref64.fm_forward(rp, fid, val, W0, V0, k)[0]
    F = len(W0)
    gW, gV, cW, cV = np.zeros(F), np.zeros((F, k)), np.zeros(F), np.zeros((F, k))
    for r in range(len(lab)):
        if w[r] == 0:
            continue
        rrp, rf, _fl, rv, rl = _row(batch, r)
        a, b, c, d = ref64.fm_grad(rrp, rf, rv, rl, W0, V0, k, pred[r:r + 1], s64[r:r + 1], l2)
        gW += w[r] * a; gV += w[r] * b; cW += w[r] * c; cV += w[r] * d
    return gW, gV, cW, cV


def ffm_weighted64(batch, W0, V0, Fc, k, pred, w, l2=L2):
    F = len(W0)
    gW, gV, cW, cV = np.zeros(F), np.zeros((F, Fc, k)), np.zeros(F), np.zeros((F, Fc, k))
    for r in range(len(w)):
        if w[r] == 0:
            continue
        rrp, rf, rfl, rv, rl = _row(batch, r)
        a, b, c, d = ref64.ffm_grad(rrp, rf, rfl, rv, rl, W0, V0, Fc, k, pred[r:r + 1], l2)
        gW += w[r] * a; gV += w[r] * b; cW += w[r] * c; cV += w[r] * d
    return gW, gV, cW, cV


def nfm_weighted_dz(z, wide, layers, label, w):
    """dz of NFM's one-hidden-layer sigmoid chain with the output delta clip(w (p - y)), in float64"""
    (w0, b0), (w1, b1) = [(np.asarray(a, np.float64).reshape(len(b), -1), np.asarray(b, np.float64)) for a, b in layers]
    o = 1.0 / (1.0 + np.exp(-(np.asarray(z, np.float64) @ w0.T + b0)))
    p = ref64.sigmoid(np.asarray(wide, np.float64) + (o @ w1.T + b1)[:, 0])
    delta = np.clip(np.asarray(w, np.float64) * (p - np.asarray(label, np.float64)), -15, 15)[:, None]
    hid = np.clip((delta @ w1) * o * (1 - o), -15, 15)
    return hid @ w0, p


def nfm_weighted64(batch, W0, V0, k, layers, pred, w, l2=L2):
    rp, fid, fld, val, lab = batch
    z, wide, s64, z_c, w_c = ref64.nfm_forward(rp, fid, val, W0, V0, k)
    _p, _dz, dz_c, _lc = ref64.nfm_head(z, wide, layers, 0, None, lab, z_c, w_c)
    dz, _p64 = nfm_weighted_dz(z, wide, layers, lab, w)
    F = len(W0)
    gW, gV, cW, cV = np.zeros(F), np.zeros((F, k)), np.zeros(F), np.zeros((F, k))
    for r in range(len(lab)):
        if w[r] == 0:
            continue
        rrp, rf, _fl, rv, rl = _row(batch, r)
        # the wide head w (p - y) and the weighted l2 enter linearly; dz already carries the weight (and its clip)
        a, b, c, d = ref64.nfm_grad(rrp, rf, rv, rl, W0, V0, k, pred[r:r + 1], s64[r:r + 1], dz[r:r + 1] / w[r], l2,
                                    dz_cond=dz_c[r:r + 1])
        gW += w[r] * a; gV += w[r] * b; cW += w[r] * c; cV += w[r] * d
    return gW, gV, cW, cV


def _nfm_layers(seed, k, H=NFM_H):
    rng = np.random.default_rng(seed)
    return [((rng.random((H, k)) - 0.5).astype(np.float32), (rng.standard_normal(H) * 0.1).astype(np.float32)),
            ((rng.random((1, H)) - 0.5).astype(np.float32), (rng.standard_normal(1) * 0.1).astype(np.float32))]


def _probe(ctx, batch, W0, V0, w, Fc=0):
    _upload(ctx, 0, batch, Fc)
    ctx.set_row_weights(0, w)
    ctx.upload_params(W0, V0)
    loss, acc = ctx.train_step(0)
    W1, V1 = ctx.download_params()
    return W1, V1, ctx.download_pred(0), loss, acc


def _check_stats(p64, lab, w, loss, acc, rtol=1e-4):
    """loss = sum w loss(p64) and acc = sum w [correct(p64)] of the float64 head p64; rows whose p64 lies within rtol of
    0.5 may count either way"""
    p = np.asarray(p64, np.float64)
    y = np.asarray(lab, np.float64)
    l64 = np.where(y == 1, -np.log(p), -np.log(1.0 - p))
    c64 = ((p > 0.5) & (y == 1)) | ((p < 0.5) & (y == 0))
    near = np.abs(p - 0.5) <= rtol
    assert abs(loss - np.sum(w * l64)) <= rtol * np.sum(w * np.abs(l64)) + 1e-5, (loss, np.sum(w * l64))
    assert abs(acc - np.sum(w * c64)) <= np.sum(w[near]) + 1e-5 * np.sum(w) + 1e-5, (acc, np.sum(w * c64))


# ------------------------------------------------------------------------------------------------------------------------
# 1. the weighted gradient against float64 on every weighted path
# ------------------------------------------------------------------------------------------------------------------------
FM_PATHS = [pytest.param(k, det, id=f"{name}-K{k}") for k, det, name in (
    (4, 0, "compact"), (8, 0, "compact"), (16, 0, "compact"), (32, 0, "compact"), (12, 0, "dense"), (3, 0, "dense"),
    (8, 1, "feature-major"), (12, 1, "feature-major"), (4, 2, "device-grouped"), (16, 2, "device-grouped"))]


@pytest.mark.parametrize("k,det", FM_PATHS)
def test_fm_weighted_gradient_vs_ref64(k, det):
    from lightctr_b200 import capi
    F = 4000
    batch = make_batch(7000 + k, F, with_val=k % 2 == 0)
    W0, V0 = make_params(7000 + k, F, k)
    w = _weights(len(batch[4]), 7100 + k)
    ctx = _ctx(capi.MODEL_FM, F, k, deterministic=det, csc_row_block=len(w) if det == 1 else 0)
    W1, V1, pred, loss, acc = _probe(ctx, batch, W0, V0, w)
    ctx.close()
    gW, gV, cW, cV = fm_weighted64(batch, W0, V0, k, pred, w)
    _check_grad("W", W0, W1, gW, cW)
    _check_grad("V", V0, V1, gV, cV)
    _check_stats(ref64.fm_forward(batch[0], batch[1], batch[3], W0, V0, k)[2], batch[4], w, loss, acc)


@pytest.mark.parametrize("k,det,prec,umma", [pytest.param(8, 0, 0, "", id="compact-MODE3-K8-fp32"),
                                             pytest.param(16, 0, 0, "", id="compact-MODE3-K16-fp32"),
                                             pytest.param(12, 1, 0, "", id="feature-major-K12-fp32"),
                                             pytest.param(12, 0, 0, "", id="dense-K12-fp32"),
                                             pytest.param(16, 0, 1, "1", id="compact-K16-bf16-nfm_mlp_umma_kernel"),
                                             pytest.param(16, 0, 1, "0", id="compact-K16-bf16-nfm_mlp_fused_kernel")])
def test_nfm_weighted_gradient_vs_ref64(k, det, prec, umma, monkeypatch):
    """row 5 carries a weight that takes its output delta past the +-15 clip.  bf16 dense layers (one hidden layer of 64,
    which the wgmma kernel takes; LCTR_MLP_UMMA=0 forces the mma.sync kernel) are held to the float64 head at 3e-2 of the
    condition figure instead of 1e-5: their operands are rounded to bf16 (8 bits)"""
    from lightctr_b200 import capi
    if umma:
        monkeypatch.setenv("LCTR_MLP_UMMA", umma)  # read when the context prepares its dense layers
    F = 4000
    H = 64 if prec else NFM_H
    rtol = 3e-2 if prec else 1e-5
    batch = make_batch(7300 + k, F, with_val=True)
    rows = len(batch[4])
    W0, V0 = make_params(7300 + k, F, k)
    layers = _nfm_layers(7300 + k, k, H)
    w = _weights(rows, 7400 + k)
    w[5] = 1000.0
    ctx = _ctx(capi.MODEL_NFM, F, k, hidden=(H,), deterministic=det, csc_row_block=rows if det else 0, mlp_precision=prec)
    for l, (a, b) in enumerate(layers):
        ctx.mlp_upload(l, a, b)
    W1, V1, pred, loss, acc = _probe(ctx, batch, W0, V0, w)
    ctx.close()
    z, wide = ref64.nfm_forward(batch[0], batch[1], batch[3], W0, V0, k)[:2]
    _dz, p64 = nfm_weighted_dz(z, wide, layers, batch[4], w)
    assert abs(w[5] * (p64[5] - batch[4][5])) > 15, "row 5 must cross the clip"
    gW, gV, cW, cV = nfm_weighted64(batch, W0, V0, k, layers, pred, w)
    _check_grad("W", W0, W1, gW, cW, rtol)
    _check_grad("V", V0, V1, gV, cV, rtol)
    _check_stats(p64, batch[4], w, loss, acc, 1e-4 if not prec else 2e-2)


def ffm_probe(Fc, k, det):
    """one weighted unit SGD step of FFM: (batch, W0, V0, w, W1, V1, pred, loss, acc)"""
    from lightctr_b200 import capi
    F = 4000
    batch = make_batch(7500 + Fc, F, rows=200, Fc=Fc, with_val=True)
    W0, V0 = make_params(7500 + Fc, F, k, Fc)
    w = _weights(len(batch[4]), 7600 + Fc)
    ctx = _ctx(capi.MODEL_FFM, F, k, Fc, deterministic=det)
    W1, V1, pred, loss, acc = _probe(ctx, batch, W0, V0, w, Fc)
    ctx.close()
    return batch, W0, V0, w, W1, V1, pred, loss, acc


FFM_KERNELS = [pytest.param(8, 4, 0, {}, id="ffm_warp_kernel-Fc8-K4"),
               pytest.param(16, 8, 0, {}, id="ffm_warp_kernel-Fc16-K8"),
               pytest.param(10, 4, 1, {}, id="ffm_warp_kernel-Fc10-K4-det1"),
               pytest.param(7, 3, 0, {}, id="ffm_fused_kernel-VEC1-Fc7-K3"),
               pytest.param(13, 6, 0, {}, id="ffm_fused_kernel-VEC2-Fc13-K6"),
               pytest.param(39, 4, 0, {"LCTR_FFM_WARP": "0"}, id="ffm_fused_kernel-VEC4-Fc39-K4"),
               pytest.param(39, 4, 0, {"LCTR_FFM_BULK": "1"}, id="ffm_fused_kernel-VEC4-bulk-Fc39-K4"),
               pytest.param(39, 4, 0, {"LCTR_FFM_TMA": "1", "LCTR_FFM_WARP": "0"}, id="ffm_tma_kernel-Fc39-K4"),
               pytest.param(12, 4, 2, {}, id="ffm_grouped-Fc12-K4")]


@pytest.mark.parametrize("Fc,k,det,env", FFM_KERNELS)
def test_ffm_weighted_gradient_vs_ref64(tmp_path, Fc, k, det, env):
    """the kernels chosen by an environment variable (read once per process) run in a process of their own"""
    if env:
        dst = str(tmp_path / "out.npz")
        code = ("import sys, numpy as np; sys.path.insert(0, %r); import test_row_weights_gpu as t; "
                "b, W0, V0, w, W1, V1, p, l, a = t.ffm_probe(%d, %d, %d); "
                "np.savez(%r, rp=b[0], fid=b[1], fld=b[2], val=b[3], lab=b[4], W0=W0, V0=V0, w=w, W1=W1, V1=V1, p=p, "
                "la=np.array([l, a]))") % (os.path.dirname(os.path.abspath(__file__)), Fc, k, det, dst)
        r = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, **env), stdout=subprocess.PIPE,
                           stderr=subprocess.STDOUT, text=True, timeout=600)
        assert r.returncode == 0, r.stdout
        with np.load(dst) as z:
            batch = (z["rp"], z["fid"], z["fld"], z["val"], z["lab"])
            W0, V0, w, W1, V1, pred = z["W0"], z["V0"], z["w"], z["W1"], z["V1"], z["p"]
            loss, acc = z["la"]
    else:
        batch, W0, V0, w, W1, V1, pred, loss, acc = ffm_probe(Fc, k, det)
    gW, gV, cW, cV = ffm_weighted64(batch, W0, V0, Fc, k, pred, w)
    _check_grad("W", W0, W1, gW, cW)
    _check_grad("V", V0, V1, gV, cV)
    p64 = ref64.ffm_forward(batch[0], batch[1], batch[2], batch[3], W0, V0, Fc, k)[1]
    _check_stats(p64, batch[4], w, loss, acc)


# ------------------------------------------------------------------------------------------------------------------------
# 2. w = 1 is the unweighted step; 3. zero weights are absent rows; 4. integer weights are duplicated rows
# ------------------------------------------------------------------------------------------------------------------------
def _train(model, F, k, batch, w, det, steps=2, opt=None, mb=0, Fc=0, hidden=()):
    from lightctr_b200 import capi
    rows = len(batch[4])
    ctx = capi.Context(getattr(capi, "MODEL_" + model), F, k, Fc, optimizer=capi.OPT_ADAGRAD if opt is None else opt, deterministic=det,
                       csc_row_block=rows if det == 1 else 0, minibatch_size=mb, l2=L2, hidden=hidden)
    if hidden:
        for l, (a, b) in enumerate(_nfm_layers(11, k)):
            ctx.mlp_upload(l, a, b)
    W0, V0 = make_params(3, F, k, Fc)
    ctx.upload_params(W0, V0)
    _upload(ctx, 0, batch, Fc)
    stats = []
    for _ in range(steps):
        if w is not None:
            ctx.set_row_weights(0, w)
        stats.append(ctx.train_step(0))
    W, V = ctx.download_params()
    s1, s2 = ctx.download_opt_state()
    pred = ctx.download_pred(0)
    ctx.close()
    return W, V, s1, s2, pred, stats


@pytest.mark.parametrize("model,k,det,Fc", [pytest.param("FM", 8, 1, 0, id="fm-det1"), pytest.param("NFM", 12, 1, 0, id="nfm-det1"),
                                           pytest.param("FM", 8, 2, 0, id="fm-det2"),
                                           pytest.param("FFM", 4, 2, 12, id="ffm-grouped-det2")])
def test_unit_weights_bit_for_bit(model, k, det, Fc):
    batch = make_batch(8000 + k, 3000, Fc=Fc, with_val=True)
    hidden = (NFM_H,) if model == "NFM" else ()
    a = _train(model, 3000, k, batch, None, det, hidden=hidden, Fc=Fc)
    b = _train(model, 3000, k, batch, np.ones(len(batch[4]), np.float32), det, hidden=hidden, Fc=Fc)
    for x, y in zip(a[:5], b[:5]):
        assert np.array_equal(x, y)
    for (l1, c1), (l2, c2) in zip(a[5], b[5]):
        assert abs(l1 - l2) <= 1e-6 * abs(l1) and c1 == c2


@pytest.mark.parametrize("model,k,Fc", [pytest.param("FM", 16, 0, id="fm-compact"), pytest.param("FM", 12, 0, id="fm-dense"),
                                        pytest.param("FFM", 4, 8, id="ffm-warp")])
def test_unit_weights_order_free(model, k, Fc):
    batch = make_batch(8100 + k, 3000, rows=200, Fc=Fc, with_val=True)
    a = _train(model, 3000, k, batch, None, 0, Fc=Fc)
    b = _train(model, 3000, k, batch, np.ones(len(batch[4]), np.float32), 0, Fc=Fc)
    for x, y in zip(a[:4], b[:4]):
        np.testing.assert_allclose(x, y, rtol=1e-5, atol=1e-6)
    for (l1, c1), (l2, c2) in zip(a[5], b[5]):
        assert abs(l1 - l2) <= 1e-5 * abs(l1) and c1 == c2


def _drop_rows(batch, keep):
    rp, fid, fld, val, lab = batch
    parts = [np.arange(rp[r], rp[r + 1]) for r in keep]
    idx = np.concatenate(parts) if parts else np.zeros(0, np.int64)
    lens = np.array([rp[r + 1] - rp[r] for r in keep], np.int64)
    return (np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), fid[idx], fld[idx], None if val is None else val[idx],
            lab[keep])


@pytest.mark.parametrize("det,model,Fc", [pytest.param(1, "FM", 0, id="fm-det1"), pytest.param(2, "FM", 0, id="fm-det2"),
                                          pytest.param(2, "FFM", 12, id="ffm-grouped-det2")])
@pytest.mark.parametrize("rule", ["ADAGRAD", "FTRL", "ADAM", "RMSPROP", "ADADELTA", "PS_SGD", "PS_ADAGRAD", "PS_DCASGD",
                                  "PS_DCASGDA"])
def test_zero_weights_are_absent_rows(rule, det, model, Fc):
    """deterministic = 1 and 2 with a fixed minibatch_size: the slot with zero-weight rows trains bit for bit as the batch
    without them; features met only by those rows keep parameters and state"""
    from lightctr_b200 import capi
    batch = make_batch(8200, 3000, Fc=Fc, with_val=True)
    rows = len(batch[4])
    w = np.ones(rows, np.float32)
    zero = np.arange(3, rows, 7)
    w[zero] = 0.0
    keep = np.setdiff1d(np.arange(rows), zero)
    opt = getattr(capi, "OPT_" + rule)
    k = 4 if Fc else 8
    a = _train(model, 3000, k, batch, w, det, opt=opt, mb=rows, Fc=Fc)
    b = _train(model, 3000, k, _drop_rows(batch, keep), None, det, opt=opt, mb=rows, Fc=Fc)
    for x, y in zip(a[:4], b[:4]):
        assert np.array_equal(x, y)
    assert np.array_equal(a[4][keep], b[4])


def test_integer_weights_are_duplicated_rows():
    batch = make_batch(8300, 3000, rows=120, with_val=True)
    rows = len(batch[4])
    w = np.random.default_rng(1).integers(0, 4, rows).astype(np.float32)
    dup = np.repeat(np.arange(rows), w.astype(np.int64))
    a = _train("FM", 3000, 8, batch, w, 1, steps=1, mb=rows)
    b = _train("FM", 3000, 8, _drop_rows(batch, dup), None, 1, steps=1, mb=rows)
    for x, y in zip(a[:4], b[:4]):
        np.testing.assert_allclose(x, y, rtol=2e-5, atol=1e-6)
    assert abs(a[5][0][0] - b[5][0][0]) <= 1e-5 * abs(b[5][0][0]) and a[5][0][1] == b[5][0][1]


# ------------------------------------------------------------------------------------------------------------------------
# 6. lifecycle
# ------------------------------------------------------------------------------------------------------------------------
def test_uploads_and_null_drop_weights():
    from lightctr_b200 import capi
    batch = make_batch(8400, 3000, with_val=True)
    rows = len(batch[4])
    w = _weights(rows, 1)
    plain = _train("FM", 3000, 8, batch, None, 1, steps=1)
    for how in ("reupload", "null", "libffm"):
        ctx = capi.Context(capi.MODEL_FM, 3000, 8, deterministic=1, csc_row_block=rows, l2=L2)
        W0, V0 = make_params(3, 3000, 8)
        ctx.upload_params(W0, V0)
        _upload(ctx, 0, batch)
        ctx.set_row_weights(0, w)
        if how == "reupload":
            _upload(ctx, 0, batch)
        elif how == "null":
            ctx.set_row_weights(0, None)
        else:
            ctx.close()
            ctx = capi.Context(capi.MODEL_FM, 3000, 8, l2=L2)
            ctx.upload_params(W0, V0)
            _upload(ctx, 0, batch)
            ctx.set_row_weights(0, w)
            text = "".join("%d %s\n" % (batch[4][r], " ".join("0:%d:1" % f for f in batch[1][batch[0][r]:batch[0][r + 1]]))
                           for r in range(rows)).encode()
            ctx.upload_libffm(0, text)
            loss = ctx.train_step(0)[0]
            ref = capi.Context(capi.MODEL_FM, 3000, 8, l2=L2)
            ref.upload_params(W0, V0)
            ref.upload_libffm(0, text)
            assert loss == ref.train_step(0)[0]
            ref.close()
            ctx.close()
            continue
        ctx.train_step(0)
        W, V = ctx.download_params()
        ctx.close()
        assert np.array_equal(W, plain[0]) and np.array_equal(V, plain[1]), how


def test_refusals_write_nothing():
    from lightctr_b200 import capi
    batch = make_batch(8500, 3000, rows=50, with_val=True)
    ctx = capi.Context(capi.MODEL_FM, 3000, 8, l2=L2)
    with pytest.raises(capi.LctrError, match="holds no rows"):
        ctx.set_row_weights(0, np.ones(50, np.float32))
    _upload(ctx, 0, batch)
    good = np.ones(50, np.float32)
    ctx.set_row_weights(0, good * 2)
    for bad, msg in ((np.full(50, -1.0), "finite"), (np.full(50, np.nan), "finite"), (np.full(50, np.inf), "finite"),
                     (np.ones(49), "49 weights")):
        with pytest.raises(capi.LctrError, match=msg):
            ctx.set_row_weights(0, bad)
    with pytest.raises(capi.LctrError, match="out of range"):
        ctx.set_row_weights(9, good)
    # the refused calls left the weights of the last good call in place
    ref = capi.Context(capi.MODEL_FM, 3000, 8, l2=L2)
    _upload(ref, 0, batch)
    ref.set_row_weights(0, good * 2)
    W0, V0 = make_params(3, 3000, 8)
    for c in (ctx, ref):
        c.upload_params(W0, V0)
    la, lb = ctx.train_step(0)[0], ref.train_step(0)[0]
    assert abs(la - lb) <= 1e-6 * abs(lb)
    ctx.close(); ref.close()


def test_score_ignores_weights():
    from lightctr_b200 import capi
    batch = make_batch(8600, 3000, rows=80, with_val=True)
    ctx = capi.Context(capi.MODEL_FM, 3000, 16, l2=L2)
    W0, V0 = make_params(3, 3000, 16)
    ctx.upload_params(W0, V0)
    _upload(ctx, 0, batch)
    a = ctx.score(0)
    ctx.set_row_weights(0, _weights(80, 2))
    assert np.array_equal(a, ctx.score(0))
    ctx.close()


def test_keyed_admission_keeps_rows_aligned():
    """admission drops entries, never rows: a weighted step on the keyed slot equals the weighted step of a dense-id
    context holding the same rows, parameters and kept entries"""
    from lightctr_b200 import capi
    batch = make_batch(8800, 3000, rows=60, with_val=False)
    rp, fid, _fld, _val, lab = batch
    keys = fid.astype(np.uint64) * np.uint64(0x9E3779B97F4A7C15)
    w = _weights(60, 3)
    cap = 4000
    ctx = capi.Context(capi.MODEL_FM, cap, 8, key_mode=capi.KEYS_HASHED, l2=L2, minibatch_size=60)
    ctx.set_key_admission(2)
    ctx.upload_batch_keys(0, rp[:31], keys[:rp[30]], None, None, lab[:30])  # the first 30 rows' keys are met once
    ctx.upload_batch_keys(0, rp, keys, None, None, lab)
    assert ctx.key_admission_stats()[0] > 0, "admission must have dropped entries"
    krp, kfid, _f, _v, klab = ctx.download_batch(0)
    assert len(krp) == 61 and len(kfid) < len(fid)
    W0, V0 = ctx.download_params()
    ctx.set_row_weights(0, w)
    kl, ka = ctx.train_step(0)
    W1, V1 = ctx.download_params()
    ctx.close()
    ref = capi.Context(capi.MODEL_FM, len(W0), 8, l2=L2, minibatch_size=60)
    ref.upload_params(W0, V0)
    ref.upload_batch(0, krp, kfid, None, None, klab.astype(np.int32))
    ref.set_row_weights(0, w)
    rl, ra = ref.train_step(0)
    RW1, RV1 = ref.download_params()
    ref.close()
    assert abs(kl - rl) <= 1e-6 * abs(rl) and ka == ra
    np.testing.assert_allclose(W1, RW1, rtol=1e-5, atol=1e-7)
    np.testing.assert_allclose(V1, RV1, rtol=1e-5, atol=1e-7)
    assert np.any(W1 != W0), "the step must move parameters"


def test_wide_and_deep_integer_weights_are_duplicated_rows():
    """Wide&Deep (wnd_backward_kernel, the fp32 dense layers' weighted delta): integer weights equal duplicated rows, zero
    weights absent rows, with a fixed minibatch_size, to the order-free tolerance"""
    import multirank as mr
    F, k, rows = 20000, 4, 128
    rp, fid, fld, lab = mr.train_batches(F, rows, 1, 0)[0]
    w = np.random.default_rng(4).integers(0, 4, rows).astype(np.float32)
    dup = np.repeat(np.arange(rows), w.astype(np.int64))
    d = _drop_rows((rp, fid, fld, None, lab), dup)
    res = []
    for batch, weights in (((rp, fid, fld, lab), w), ((d[0], d[1], d[2], d[4]), None)):
        ctx = mr.make_context("wnd", F, k, 0, 1, minibatch_size=rows, max_nnz=rows * 400)
        ctx.upload_params(*mr.make_params(F, k, "wnd"))
        for l, (a, b) in enumerate(mr.dense_layers("wnd", k)):
            ctx.mlp_upload(l, a, b)
        mr.upload(ctx, "wnd", 0, batch)
        if weights is not None:
            ctx.set_row_weights(0, weights)
        loss, acc = ctx.train_step(0)
        W, V = ctx.download_params()
        dims = mr.layer_dims("wnd", k)
        mlp = [ctx.mlp_download(l, dims[l], dims[l + 1]) for l in range(len(dims) - 1)]
        ctx.close()
        res.append((loss, acc, W, V, mlp))
    (l1, a1, W1, V1, m1), (l2, a2, W2, V2, m2) = res
    assert abs(l1 - l2) <= 1e-5 * abs(l2) and a1 == a2
    np.testing.assert_allclose(W1, W2, rtol=1e-4, atol=1e-6)
    np.testing.assert_allclose(V1, V2, rtol=1e-4, atol=1e-6)
    for (x1, y1), (x2, y2) in zip(m1, m2):
        np.testing.assert_allclose(x1, x2, rtol=1e-4, atol=1e-6)
        np.testing.assert_allclose(y1, y2, rtol=1e-4, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------------------
# two ranks on one GPU: each rank weights its own rows; dist.cu carries the weighted gradients unchanged
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,k", [("fm", 16), ("fm", 12), ("ffm", 4), ("nfm", 16)],
                         ids=["fm-compact", "fm-dense", "ffm", "nfm"])
def test_two_ranks_weighted_equal_world1(tmp_path, model, k):
    """parameters and the ranks' summed (loss, acc) equal a world-1 context trained on multirank.global_batch with the
    concatenated weights, to the two-rank tolerance (the sparse scatter sums in arbitrary order)"""
    import dist_weights_worker as wk
    import multirank as mr
    from lightctr_b200 import dist as ldist
    F, rows = 20000, 256
    out = str(tmp_path)
    mr.launch("dist_weights_worker.py", out, ["--model", model, "--k", str(k), "--F", str(F), "--rows", str(rows)])
    parts, res = mr.load(out), mr.load_json(out)
    ctx = mr.make_context(model, F, k, 0, 1, minibatch_size=2 * rows, max_nnz=rows * 400)
    ctx.upload_params(*mr.make_params(F, k, model))
    for l, (w, b) in enumerate(mr.dense_layers(model, k)):
        ctx.mlp_upload(l, w, b)
    per_rank = [mr.train_batches(F, rows, wk.STEPS, r) for r in range(2)]
    for i in range(wk.STEPS):
        g = mr.global_batch([per_rank[r][i] for r in range(2)])
        mr.upload(ctx, model, 0, g)
        ctx.set_row_weights(0, np.concatenate([wk.weights(r, i, len(per_rank[r][i][3])) for r in range(2)]))
        loss, acc = ctx.train_step(0)
        got_l = sum(res[r]["loss"][i] for r in range(2))
        got_a = sum(res[r]["acc"][i] for r in range(2))
        assert abs(got_l - loss) <= 1e-5 * abs(loss), (i, got_l, loss)
        assert abs(got_a - acc) <= 1e-5 * abs(acc) + 1e-3, (i, got_a, acc)
    W, V = ctx.download_params()
    ctx.close()
    assert np.max(np.abs(ldist.merge_shards([p["W"] for p in parts], 2, F) - W)) < 1e-5
    assert np.max(np.abs(ldist.merge_shards([p["V"] for p in parts], 2, F) - V)) < 1e-5
