"""NFM dense layers in tensor-core mode (mlp_precision = BF16, lightctr_b200/csrc/mlp_bf16.cu).

This mode is not a 1e-5 trajectory mode: operands are rounded to bf16 (fp32 accumulation, fp32 masters).  It is checked
  (1) against a plain PyTorch fp32 emulation of Fully_Conn_Layer (fullyconnLayer.h:80-180) that rounds at exactly the
      same points (z, W, activations, deltas -> bf16), on predictions and on every dW/db (tolerances at the asserts:
      a pre-rounding difference of 1 fp32 ulp -- __expf vs expf, summation order -- can move an activation by one bf16
      ulp = 2^-8 relative, so elementwise bars are a few 1e-3 of the tensor's scale);
  (2) against the fp32 parity mode of the same library on the same inputs: first-step Adagrad updates are sign-like
      (lr * g / sqrt(g^2 + eps)), so the sign pattern of the V and MLP updates validates dz / dW end to end;
  (3) on a 12-step loss trajectory against the fp32 mode."""
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _batch(seed, rows, F, nnz_per_row):
    rng = np.random.RandomState(seed)
    cnt = rng.randint(nnz_per_row // 2, nnz_per_row + 1, size=rows)
    rp = np.zeros(rows + 1, np.int64)
    rp[1:] = np.cumsum(cnt)
    fid = np.concatenate([rng.choice(F, c, replace=False) for c in cnt]).astype(np.uint32)
    label = (rng.rand(rows) < 0.4).astype(np.int32)
    return rp, fid, label


def _params(seed, F, k, dims):
    rng = np.random.RandomState(seed)
    W = (rng.randn(F) * 0.05).astype(np.float32)
    V = (rng.randn(F * k) * 0.15).astype(np.float32)
    layers = []
    for i in range(len(dims) - 1):
        w = (rng.randn(dims[i + 1], dims[i]) * (1.5 / np.sqrt(dims[i]))).astype(np.float32)
        b = (rng.randn(dims[i + 1]) * 0.1).astype(np.float32)
        layers.append((w, b))
    return W, V, layers


def _ctx(capi, prec, F, k, hidden, act, mb, W, V, layers, masks=None, lr=0.05):
    c = capi.Context(capi.MODEL_NFM, F, k, hidden=hidden, activation=act, mlp_precision=prec, minibatch_size=mb, lr=lr)
    c.upload_params(W, V)
    for l, (w, b) in enumerate(layers):
        c.mlp_upload(l, w, b)
        if masks is not None and l < len(hidden):
            c.mlp_set_mask(l, masks[l])
    return c


def _emulate(torch, capi, rp, fid, label, W, V, k, layers, act, masks):
    """fp32 PyTorch reference with the kernel's bf16 rounding points."""
    bf = lambda x: x.to(torch.bfloat16).to(torch.float32)
    rows = len(rp) - 1
    Vt = torch.from_numpy(V.reshape(-1, k))
    z = torch.zeros(rows, k)
    wide = torch.zeros(rows)
    for r in range(rows):
        ids = torch.from_numpy(fid[rp[r]:rp[r + 1]].astype(np.int64))
        t = Vt[ids]
        s = t.sum(0)
        z[r] = 0.5 * s * s - 0.5 * (t * t).sum(0)  # train_nfm_algo.cpp:87-94
        wide[r] = torch.from_numpy(W)[ids].sum()
    y = torch.from_numpy(label.astype(np.float32))
    fwd = (lambda v: torch.sigmoid(v)) if act == capi.ACT_SIGMOID else (lambda v: torch.tanh(v))
    dact = (lambda a: a * (1 - a)) if act == capi.ACT_SIGMOID else (lambda a: 1 - a * a)
    nh = len(layers) - 1
    xs = [bf(z)]
    for l in range(nh):
        w, b = torch.from_numpy(layers[l][0]), torch.from_numpy(layers[l][1])
        pre = xs[l] @ bf(w).T + b
        pre = pre * torch.from_numpy(masks[l])  # masked neurons: pre-activation forced to 0
        xs.append(bf(fwd(pre)))
    wl, bl = torch.from_numpy(layers[nh][0]).reshape(-1), torch.from_numpy(layers[nh][1])
    out = xs[nh] @ wl + bl
    p = torch.sigmoid(wide + out)
    d3 = (p - y).clamp(-15, 15)
    grads = [None] * (nh + 1)
    grads[nh] = ((d3[:, None] * xs[nh]).sum(0), d3.sum().reshape(1))
    delta = bf((d3[:, None] * wl[None, :] * dact(xs[nh])).clamp(-15, 15))
    dz = None
    for l in range(nh - 1, -1, -1):
        grads[l] = (delta.T @ xs[l], delta.sum(0))
        dx = (delta * torch.from_numpy(masks[l])) @ bf(torch.from_numpy(layers[l][0]))
        if l > 0:
            delta = bf((dx * dact(xs[l])).clamp(-15, 15))
        else:
            dz = dx
    return p.numpy(), [(g[0].numpy(), g[1].numpy()) for g in grads], dz.numpy()


# which kernel takes the chain: "umma" = wgmma (mlp_umma.cu: hidden widths multiples of 64, no dropout mask), "mma" = the
# mma.sync kernel of mlp_bf16.cu (everything else)
@pytest.mark.parametrize("hidden,act_name,rows,masked,kernel", [((64, 32), "sigmoid", 300, False, "mma"),
                                                                ((256, 128, 64), "sigmoid", 257, False, "umma"),
                                                                ((256, 128, 64), "tanh", 200, False, "umma"),
                                                                ((128, 64), "sigmoid", 300, False, "umma"),
                                                                ((128, 128), "tanh", 130, False, "umma"),
                                                                ((256, 128, 64), "tanh", 129, True, "mma")])
def test_bf16_mlp_matches_emulation(hidden, act_name, rows, masked, kernel, capfd, monkeypatch):
    torch = pytest.importorskip("torch")
    from lightctr_b200 import capi
    monkeypatch.setenv("LCTR_MLP_UMMA_TRACE", "1")  # the wgmma kernel reports its phase timings on stderr when it runs
    F, k = 3000, 16
    act = capi.ACT_SIGMOID if act_name == "sigmoid" else capi.ACT_TANH
    dims = [k] + list(hidden) + [1]
    rp, fid, label = _batch(3, rows, F, 24)
    W, V, layers = _params(5, F, k, dims)
    rng = np.random.RandomState(11)
    masks = [(rng.rand(h) > (0.3 if masked else -1.0)).astype(np.float32) for h in hidden]
    os.environ["LCTR_MLP_SKIP_UPDATE"] = "1"
    try:
        c = _ctx(capi, capi.MLP_BF16, F, k, hidden, act, rows, W, V, layers, masks)
    finally:
        del os.environ["LCTR_MLP_SKIP_UPDATE"]
    c.upload_batch(0, rp, fid, None, None, label)
    loss, acc = c.train_step(0)
    pred = c.download_pred(0)
    assert ("[mlp_umma trace" in capfd.readouterr().err) == (kernel == "umma")
    p_ref, g_ref, _ = _emulate(torch, capi, rp, fid, label, W, V, k, layers, act, masks)
    assert np.max(np.abs(pred - p_ref)) < 3e-3, np.max(np.abs(pred - p_ref))  # bf16-ulp flips of single activations
    y = label.astype(np.float64)
    loss_ref = float(-(y * np.log(p_ref.astype(np.float64)) + (1 - y) * np.log(1 - p_ref.astype(np.float64))).sum())
    assert abs(loss - loss_ref) < 2e-3 * abs(loss_ref), (loss, loss_ref)
    for l in range(len(dims) - 1):
        dw, db = c.mlp_download_grad(l, dims[l], dims[l + 1])
        rw, rb_ = g_ref[l]
        for got, ref, name in ((dw.reshape(rw.shape), rw, "dW"), (db, rb_, "db")):
            scale = np.max(np.abs(ref)) + 1e-12
            err = np.max(np.abs(got - ref)) / scale
            assert err < 1e-2, (l, name, err)  # max-norm relative; typical measured value is ~1e-3
            # and the bulk of the entries is much tighter than the max
            assert np.median(np.abs(got - ref)) / scale < 1e-3, (l, name)
    c.close()


def test_wgmma_and_mma_sync_kernels_agree(monkeypatch):
    """The two tensor-core kernels (mlp_umma.cu: wgmma.mma_async; mlp_bf16.cu: mma.sync) round at the same points; on the
    C4 chain they must agree to a few bf16 ulps of single activations (the sigmoid is 1/(1+2^t) on MUFU in one and
    __expf/__fdividef in the other)."""
    from lightctr_b200 import capi
    F, k, hidden, rows = 3000, 16, (256, 128, 64), 1000
    dims = [k] + list(hidden) + [1]
    rp, fid, label = _batch(21, rows, F, 24)
    W, V, layers = _params(23, F, k, dims)
    out = {}
    monkeypatch.setenv("LCTR_MLP_SKIP_UPDATE", "1")
    for flag in ("0", "1"):
        monkeypatch.setenv("LCTR_MLP_UMMA", flag)  # read when the context prepares its dense layers
        c = _ctx(capi, capi.MLP_BF16, F, k, hidden, capi.ACT_SIGMOID, rows, W, V, layers)
        c.upload_batch(0, rp, fid, None, None, label)
        loss, _ = c.train_step(0)
        out[flag] = (loss, c.download_pred(0), [c.mlp_download_grad(l, dims[l], dims[l + 1]) for l in range(len(dims) - 1)])
        c.close()
    (l0, p0, g0), (l1, p1, g1) = out["0"], out["1"]
    assert abs(l0 - l1) < 1e-3 * abs(l0), (l0, l1)
    assert np.max(np.abs(p0 - p1)) < 3e-3
    for l in range(len(dims) - 1):
        for a, b, name in ((g0[l][0], g1[l][0], "dW"), (g0[l][1], g1[l][1], "db")):
            scale = np.max(np.abs(a)) + 1e-12
            assert np.max(np.abs(a - b)) / scale < 1e-2, (l, name)
            assert np.median(np.abs(a - b)) / scale < 1e-3, (l, name)


def test_bf16_first_step_signs_match_fp32_mode():
    from lightctr_b200 import capi
    F, k, hidden, rows = 3000, 16, (128, 64), 512
    dims = [k] + list(hidden) + [1]
    rp, fid, label = _batch(7, rows, F, 24)
    W, V, layers = _params(9, F, k, dims)
    res = {}
    for prec in (capi.MLP_FP32, capi.MLP_BF16):
        c = _ctx(capi, prec, F, k, hidden, capi.ACT_SIGMOID, rows, W, V, layers)
        c.upload_batch(0, rp, fid, None, None, label)
        loss, _ = c.train_step(0)
        W1, V1 = c.download_params()
        mlp = [c.mlp_download(l, dims[l], dims[l + 1]) for l in range(len(dims) - 1)]
        res[prec] = (loss, V1 - V, [m[0] - layers[l][0].reshape(-1) for l, m in enumerate(mlp)])
        c.close()
    l32, dV32, dM32 = res[capi.MLP_FP32]
    l16, dV16, dM16 = res[capi.MLP_BF16]
    assert abs(l16 - l32) < 2e-3 * abs(l32), (l16, l32)
    lr = 0.05
    sel = np.abs(dV32) > 0.5 * lr  # coordinates whose first Adagrad step is saturated: update == -lr * sign(g)
    assert sel.sum() > 1000
    agree = np.mean(np.sign(dV32[sel]) == np.sign(dV16[sel]))
    assert agree > 0.98, agree  # dz (MLP -> embedding gradient) has the right sign pattern
    for l in range(len(dims) - 1):
        s = np.abs(dM32[l]) > 0.5 * lr
        agree = np.mean(np.sign(dM32[l][s]) == np.sign(dM16[l][s]))
        assert agree > 0.98, (l, agree)


def test_bf16_trajectory_tracks_fp32_mode():
    from lightctr_b200 import capi
    F, k, hidden, rows = 3000, 16, (256, 128, 64), 1024
    dims = [k] + list(hidden) + [1]
    rp, fid, label = _batch(13, rows, F, 24)
    W, V, layers = _params(17, F, k, dims)
    curves = {}
    for prec in (capi.MLP_FP32, capi.MLP_BF16):
        c = _ctx(capi, prec, F, k, hidden, capi.ACT_SIGMOID, 256, W, V, layers, lr=0.02)
        c.upload_batch(0, rp, fid, None, None, label)
        cur = []
        for e in range(3):
            tot = 0.0
            for b in range(0, rows, 256):  # minibatches of 256 (two 128-sample tiles each)
                tot += c.train_step(0, b, b + 256)[0]
            cur.append(tot)
        curves[prec] = cur
        c.close()
    a, b = np.array(curves[capi.MLP_FP32]), np.array(curves[capi.MLP_BF16])
    assert np.all(np.abs(a - b) < 3e-2 * np.abs(a)), (a, b)
    assert b[-1] < b[0]  # it learns
