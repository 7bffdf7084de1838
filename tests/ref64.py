"""Float64 restatement of the FM / NFM / FFM forward and per-feature gradients, written from each operation's definition
(not from any kernel's arithmetic order).  The GPU shape and gradient tests (tests/test_kernel_shapes_gpu.py,
tests/test_gradients_gpu.py) compare the CUDA kernels with it; tests/test_ref64_cpu.py holds it against the CPU oracle first.

Every function takes a CSR batch (row_ptr, fid, val; val None = all ones) and returns float64 arrays.  Next to each value
it returns a condition figure: the same expression evaluated on absolute values, so a tolerance can be stated as
`|got - want| <= rtol * cond + atol` and hold for any fp32 summation order.

nfm_head restates NFM's dense layers (forward, pCTR and the input delta dz that the embedding backward consumes), and
probe_excess is the bound of tests/test_gradients_gpu.py, which recovers each kernel's gradient from one unit SGD step.

Reference quirks kept on purpose:
- FM: gV = (sumVX - x V) * gradW + l2 V per entry, with gradW = (p - y) x + l2 W (the W regulariser leaks into gV).
- FFM: l2 V is added once per PAIR an entry takes part in, and rows whose prediction equals the label contribute nothing.
- the sigmoid clamps to 1e-7 / 1 - 1e-7 outside [-16, 16] (activations.h)."""
import numpy as np


def _rows(row_ptr):
    row_ptr = np.asarray(row_ptr, np.int64)
    return np.repeat(np.arange(len(row_ptr) - 1), np.diff(row_ptr))


def _val(val, nnz):
    return np.ones(nnz) if val is None else np.asarray(val, np.float64)


def sigmoid(z):
    z = np.asarray(z, np.float64)
    p = 1.0 / (1.0 + np.exp(-np.clip(z, -60, 60)))
    p = np.where(z < -16, float(np.float32(1e-7)), p)
    return np.where(z > 16, float(np.float32(1.0 - 1e-7)), p)


def fm_forward(row_ptr, fid, val, W, V, k):
    """FM: sumVX[r] = sum_i x_i V_i; logit = sum_i w_i x_i + 0.5 (|sumVX|^2 - sum_i |x_i V_i|^2).
    Returns (sumvx [rows, k], logit [rows], pctr [rows], sumvx_cond [rows, k], logit_cond [rows])."""
    rows = len(row_ptr) - 1
    r = _rows(row_ptr)
    f = np.asarray(fid, np.int64)
    x = _val(val, len(f))
    V2 = np.asarray(V, np.float64).reshape(-1, k)
    t = V2[f] * x[:, None]
    sumvx = np.zeros((rows, k))
    np.add.at(sumvx, r, t)
    sabs = np.zeros((rows, k))
    np.add.at(sabs, r, np.abs(t))
    wx = np.asarray(W, np.float64)[f] * x
    lin = np.bincount(r, wx, rows)
    lin_abs = np.bincount(r, np.abs(wx), rows)
    self_sq = np.bincount(r, np.sum(t * t, 1), rows)
    logit = lin + 0.5 * (np.sum(sumvx * sumvx, 1) - self_sq)
    logit_cond = lin_abs + 0.5 * (np.sum(sabs * sabs, 1) + self_sq)
    return sumvx, logit, sigmoid(logit), sabs, logit_cond


def nfm_forward(row_ptr, fid, val, W, V, k):
    """NFM embedding side: bi-interaction z[r] = 0.5 (sumVX^2 - sum_i (x_i V_i)^2) per factor, wide[r] = sum_i w_i x_i.
    Returns (z [rows, k], wide [rows], sumvx [rows, k], z_cond [rows, k], wide_cond [rows])."""
    rows = len(row_ptr) - 1
    r = _rows(row_ptr)
    f = np.asarray(fid, np.int64)
    x = _val(val, len(f))
    t = np.asarray(V, np.float64).reshape(-1, k)[f] * x[:, None]
    sumvx = np.zeros((rows, k))
    np.add.at(sumvx, r, t)
    sabs = np.zeros((rows, k))
    np.add.at(sabs, r, np.abs(t))
    sq = np.zeros((rows, k))
    np.add.at(sq, r, t * t)
    wx = np.asarray(W, np.float64)[f] * x
    return (0.5 * (sumvx * sumvx - sq), np.bincount(r, wx, rows), sumvx, 0.5 * (sabs * sabs + sq),
            np.bincount(r, np.abs(wx), rows))


def fm_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, l2):
    """Per-feature FM gradient summed over the batch: gW[f] = sum (p - y) x + l2 w_f;
    gV[f] = sum (sumVX_r - x V_f) * gradW + l2 V_f.  pred / sumvx are the forward's (rows,) / (rows, k).
    Returns (gW [F], gV [F, k], gW_cond [F], gV_cond [F, k])."""
    return _fm_like_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, l2, None)


def nfm_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, dz, l2, dz_cond=None):
    """Per-feature NFM gradient from the dense layers' input delta dz (rows, k): gW as FM;
    gV[f] = sum (sumVX_r - x V_f) * (dz_r x) + l2 V_f.  dz_cond (nfm_head's figure for dz) folds the error of a dz that
    was itself computed in fp32 into gV's condition: sum |sumVX_r - x V_f| |x| dz_cond_r."""
    return _fm_like_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, l2, dz, dz_cond)


def _act(h, act):
    """hidden activation and its derivative as a function of the output (activations.h): 0 sigmoid, 1 tanh"""
    if act == 0:
        o = 1.0 / (1.0 + np.exp(-np.clip(h, -60, 60)))
        return o, o * (1 - o), np.abs(1 - 2 * o)
    o = np.tanh(h)
    return o, 1 - o * o, 2 * np.abs(o)


def nfm_head(z, wide, layers, act, masks, label, z_cond=None, wide_cond=None):
    """The Fully_Conn_Layer chain of NFM in float64 (the oracle's orc_mlp_forward / orc_mlp_backward): layers = [(weight
    [out, in], bias [out])...], the last one linear with one output; every hidden output is masked (mask 0 -> 0) and then
    activated (masked ones included); p = sigmoid(wide + out); the delta p - y runs back with a +-15 clip per layer and the
    hidden masks on the weights, and dz is the first layer's input delta.  masks: one array per layer (None = all ones).
    z_cond / wide_cond: nfm_forward's figures for z and the wide part.
    Returns (pctr [rows], dz [rows, k], dz_cond [rows, k], logit_cond [rows]); the figures carry the fp32 rounding of
    every dot product, activation and input through the chain, so that |dz - dz64| <= 1e-5 * dz_cond for an fp32 chain."""
    a = np.asarray(z, np.float64)
    c = np.zeros_like(a) if z_cond is None else np.asarray(z_cond, np.float64)
    n = len(layers)
    acts = []  # (output, its figure, activation', |d act' / d output|) per hidden layer
    for l, (w, b) in enumerate(layers):
        w = np.asarray(w, np.float64).reshape(len(b), -1)
        b = np.asarray(b, np.float64)
        h = a @ w.T + b
        ch = c @ np.abs(w).T + np.abs(a) @ np.abs(w).T + np.abs(b)
        if l + 1 < n:
            m = np.ones(len(b)) if masks is None or masks[l] is None else np.asarray(masks[l], np.float64)
            h, ch = h * m, ch * m
            o, d1, d2 = _act(h, act)
            co = d1 * ch + np.abs(o)
            acts.append((o, co, d1, d2))
            a, c = o, co
        else:
            out, cout = h[:, 0], ch[:, 0]
    logit = np.asarray(wide, np.float64) + out
    logit_cond = (np.zeros_like(logit) if wide_cond is None else np.asarray(wide_cond, np.float64)) + cout
    p = sigmoid(logit)
    delta = np.clip(p - np.asarray(label, np.float64), -15, 15)[:, None]
    cd = (p * (1 - p) * logit_cond + np.abs(p))[:, None]
    for l in range(n - 1, -1, -1):
        w, b = layers[l]
        w = np.asarray(w, np.float64).reshape(len(b), -1)
        if l + 1 < n and masks is not None and masks[l] is not None:
            w = w * np.asarray(masks[l], np.float64)[:, None]
        delta = np.clip(delta, -15, 15)
        idl = delta @ w
        cidl = cd @ np.abs(w) + np.abs(delta) @ np.abs(w)
        if l == 0:
            return p, idl, cidl, logit_cond
        o, co, d1, d2 = acts[l - 1]
        delta = idl * d1
        cd = d1 * cidl + np.abs(idl) * d2 * co + np.abs(delta)


def probe_excess(got, want, cond, w1, rtol=1e-5):
    """The bound of a gradient recovered from one unit SGD step (g = w0 - w1, see tests/test_gradients_gpu.py):
    |g - g64| <= rtol * cond + spacing(w1).  Returns |g - g64| minus the bound, per coordinate (> 0: out of bound)."""
    err = np.abs(np.asarray(got, np.float64) - np.asarray(want, np.float64))
    return err - (rtol * np.asarray(cond, np.float64) + np.spacing(np.abs(np.asarray(w1, np.float32))).astype(np.float64))


def _fm_like_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, l2, dz, dz_cond=None):
    r = _rows(row_ptr)
    f = np.asarray(fid, np.int64)
    x = _val(val, len(f))
    W = np.asarray(W, np.float64)
    V2 = np.asarray(V, np.float64).reshape(-1, k)
    F = len(W)
    d = np.asarray(pred, np.float64) - np.asarray(label, np.float64)
    s = np.asarray(sumvx, np.float64).reshape(-1, k)
    gw = d[r] * x + l2 * W[f]
    gw_abs = np.abs(d[r] * x) + np.abs(l2 * W[f])
    tv = s[r] - x[:, None] * V2[f]
    # |sumVX_r - x V_f| is itself a cancelling sum: its condition is sum_j |x_j V_j| (with V_f counted twice)
    sabs = np.zeros_like(s)
    np.add.at(sabs, r, np.abs(V2[f] * x[:, None]))
    tv_abs = sabs[r] + np.abs(x[:, None] * V2[f])
    if dz is None:
        mult, mult_abs = gw[:, None], gw_abs[:, None]
    else:
        dzr = np.asarray(dz, np.float64).reshape(-1, k)[r]
        mult, mult_abs = dzr * x[:, None], np.abs(dzr * x[:, None])
        if dz_cond is not None:
            mult_abs = mult_abs + np.asarray(dz_cond, np.float64).reshape(-1, k)[r] * np.abs(x[:, None])
    gv = tv * mult + l2 * V2[f]
    gv_abs = tv_abs * mult_abs + np.abs(l2 * V2[f])
    gW = np.bincount(f, gw, F)
    gW_c = np.bincount(f, gw_abs, F)
    gV = np.zeros((F, k))
    gV_c = np.zeros((F, k))
    np.add.at(gV, f, gv)
    np.add.at(gV_c, f, gv_abs)
    return gW, gV, gW_c, gV_c


def _ffm_rows(row_ptr, fid, field, val):
    row_ptr = np.asarray(row_ptr, np.int64)
    f = np.asarray(fid, np.int64)
    fl = np.asarray(field, np.int64)
    x = _val(val, len(f))
    for r in range(len(row_ptr) - 1):
        b, e = row_ptr[r], row_ptr[r + 1]
        yield r, f[b:e], fl[b:e], x[b:e]


def ffm_forward(row_ptr, fid, field, val, W, V, Fc, k):
    """FFM by the O(n^2) pair loop: logit = sum_i w_i x_i + sum_{i<j} <V[f_i, fl_j], V[f_j, fl_i]> x_i x_j.
    Returns (logit [rows], pctr [rows], logit_cond [rows])."""
    rows = len(row_ptr) - 1
    W = np.asarray(W, np.float64)
    V3 = np.asarray(V, np.float64).reshape(-1, Fc, k)
    logit, cond = np.zeros(rows), np.zeros(rows)
    for r, f, fl, x in _ffm_rows(row_ptr, fid, field, val):
        n = len(f)
        if n == 0:
            continue
        A = V3[f[:, None], fl[None, :]]                      # A[i, j] = V[f_i, fl_j]
        prod = A * np.transpose(A, (1, 0, 2))                 # V[f_i, fl_j] * V[f_j, fl_i]
        P = prod.sum(2) * x[:, None] * x[None, :]
        Pa = np.abs(prod).sum(2) * np.abs(x[:, None] * x[None, :])
        iu = np.triu_indices(n, 1)
        logit[r] = np.sum(W[f] * x) + P[iu].sum()
        cond[r] = np.sum(np.abs(W[f] * x)) + Pa[iu].sum()
    return logit, sigmoid(logit), cond


def ffm_grad(row_ptr, fid, field, val, label, W, V, Fc, k, pred, l2):
    """Per-feature FFM gradient: gW[f] = sum (p - y) x + l2 w_f; for each pair i < j of a row, with s = (p - y) x_i x_j,
    gV[f_i, fl_j] += s V[f_j, fl_i] + l2 V[f_i, fl_j] and gV[f_j, fl_i] += s V[f_i, fl_j] + l2 V[f_j, fl_i].  Rows whose
    prediction equals their label are skipped entirely.  Returns (gW [F], gV [F, Fc, k], gW_cond, gV_cond)."""
    W = np.asarray(W, np.float64)
    V3 = np.asarray(V, np.float64).reshape(-1, Fc, k)
    F = len(W)
    gW, gWc = np.zeros(F), np.zeros(F)
    gV, gVc = np.zeros((F, Fc, k)), np.zeros((F, Fc, k))
    pred = np.asarray(pred, np.float64)
    label = np.asarray(label, np.float64)
    for r, f, fl, x in _ffm_rows(row_ptr, fid, field, val):
        d = pred[r] - label[r]
        if d == 0 or len(f) == 0:
            continue
        np.add.at(gW, f, d * x + l2 * W[f])
        np.add.at(gWc, f, np.abs(d * x) + np.abs(l2 * W[f]))
        n = len(f)
        i, j = np.triu_indices(n, 1)
        s = (d * x[i] * x[j])[:, None]
        vi, vj = V3[f[i], fl[j]], V3[f[j], fl[i]]            # V[f_i, fl_j], V[f_j, fl_i]
        np.add.at(gV, (f[i], fl[j]), s * vj + l2 * vi)
        np.add.at(gV, (f[j], fl[i]), s * vi + l2 * vj)
        np.add.at(gVc, (f[i], fl[j]), np.abs(s * vj) + np.abs(l2 * vi))
        np.add.at(gVc, (f[j], fl[i]), np.abs(s * vi) + np.abs(l2 * vj))
        # the partners of entry i in its own field a_i form a sum of x_j V[f_j, a_i] that a kernel may take as the field's
        # whole sum minus x_i V[f_i, a_i] (the cancelling form of FM's sumVX - x V): that term counts in the condition
        own = np.bincount(fl, minlength=V3.shape[1])[fl] > 1
        np.add.at(gVc, (f[own], fl[own]), np.abs(d * x[own] ** 2)[:, None] * np.abs(V3[f[own], fl[own]]))
    return gW, gV, gWc, gVc
