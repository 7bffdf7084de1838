"""Float64 restatement of the FM / NFM / FFM forward and per-feature gradients, written from each operation's definition
(not from any kernel's arithmetic order).  The GPU shape tests (tests/test_kernel_shapes_gpu.py) compare the CUDA kernels
with it; tests/test_ref64_cpu.py holds it against the CPU oracle first.

Every function takes a CSR batch (row_ptr, fid, val; val None = all ones) and returns float64 arrays.  Next to each value
it returns a condition figure: the same expression evaluated on absolute values, so a tolerance can be stated as
`|got - want| <= rtol * cond + atol` and hold for any fp32 summation order.

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


def nfm_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, dz, l2):
    """Per-feature NFM gradient from the dense layers' input delta dz (rows, k): gW as FM;
    gV[f] = sum (sumVX_r - x V_f) * (dz_r x) + l2 V_f."""
    return _fm_like_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, l2, dz)


def _fm_like_grad(row_ptr, fid, val, label, W, V, k, pred, sumvx, l2, dz):
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
    return gW, gV, gWc, gVc
