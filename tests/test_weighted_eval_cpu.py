"""Weighted test-set metrics and weighted streamed batches without a GPU: the numpy restatement of the weighted metrics'
rule (tests/weighted_eval.py) against the unweighted walk, and the new symbols and their bindings."""
import ctypes as C
import os

import numpy as np

import weighted_eval as we
from conftest import ROOT


def _data(n, seed, ties=False):
    rng = np.random.default_rng(seed)
    p = rng.random(n).astype(np.float32)
    if ties:  # saturated predictions and a handful of distinct values: many rows per bucket
        p = rng.choice(np.array([0.0, 1.0, 0.25, 0.5, 0.75], np.float32), n)
    y = (rng.random(n) < 0.3).astype(np.int32)
    return p, y


def _bits(x):
    return np.float32(x).view(np.uint32)


def test_unit_weights_are_the_unweighted_walk():
    for seed, ties in ((1, False), (2, True)):
        p, y = _data(20000, seed, ties)
        lw, cw, aw = we.eval_weighted(p, y, np.ones(len(p), np.float32))
        lu, cu, au = we.eval_unweighted(p, y)
        assert _bits(lw) == _bits(lu) and cw == float(cu) and _bits(aw) == _bits(au), (seed, lw, lu, cw, cu, aw, au)


def test_integer_weights_are_duplicated_rows():
    for seed, ties in ((3, False), (4, True)):
        p, y = _data(5000, seed, ties)
        w = np.random.default_rng(seed).integers(0, 6, len(p)).astype(np.float32)
        _l, cw, aw = we.eval_weighted(p, y, w)
        rows = np.repeat(np.arange(len(p)), w.astype(np.int64))
        _l2, cu, au = we.eval_unweighted(p[rows], y[rows])
        assert cw == float(cu) and _bits(aw) == _bits(au), (seed, cw, cu, aw, au)


def test_power_of_two_scale_keeps_the_auc():
    p, y = _data(20000, 5)
    w = (0.5 + 3.5 * np.random.default_rng(5).random(len(p))).astype(np.float32)
    a0 = we.eval_weighted(p, y, w)[2]
    for k in (-100, -7, 1, 30, 120):
        a = we.eval_weighted(p, y, np.ldexp(w, k).astype(np.float32))[2]
        assert _bits(a) == _bits(a0), (k, a, a0)


def test_tiny_weights_leave_the_auc_alone():
    """a weight below 2^(E-33) rounds to q = 0: the AUC is that of the other rows, the loss and correct still count it"""
    p, y = _data(4000, 6)
    w = np.ones(len(p), np.float32)
    w[::5] = 2.0 ** -40
    _l, c, a = we.eval_weighted(p, y, w)
    keep = w == 1.0
    assert we.fixed_point(w)[~keep].max() == 0
    _lk, ck, ak = we.eval_unweighted(p[keep], y[keep])
    assert _bits(a) == _bits(ak)
    assert c > ck  # the tiny rows' 2^-40 each are above the spacing of the double sum


def test_zero_weights_and_no_positives_give_auc_zero():
    p, y = _data(1000, 7)
    assert we.eval_weighted(p, y, np.zeros(len(p), np.float32)) == (np.float32(0), 0.0, np.float32(0))
    assert we.eval_weighted(p, np.ones(len(p), np.int32), np.ones(len(p), np.float32))[2] == 0


def test_symbols_exported_and_bound():
    from lightctr_b200 import build, capi
    names = ("lctr_eval_weighted", "lctr_eval_pred_weighted", "lctr_train_batch_weighted_async")
    L = C.CDLL(build.build())
    for n in names:
        assert n in capi.SYMBOLS and hasattr(L, n), n
    L = capi.load_library()
    vp, f32p, d = C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_double)
    assert L.lctr_eval_weighted.argtypes == [vp, C.c_int, f32p, d, f32p]
    assert L.lctr_eval_pred_weighted.argtypes == [vp, C.c_int64, vp, vp, vp, f32p, d, f32p]
    assert L.lctr_train_batch_weighted_async.argtypes == [vp, C.c_int64, C.c_int64, vp, vp, vp, vp, vp, vp,
                                                          C.POINTER(C.c_uint64)]
    hdr = " ".join(open(os.path.join(ROOT, "include", "lightctr_b200.h")).read().split())
    for decl in ("int lctr_eval_weighted(lctr_ctx* ctx, int slot, float* loss_sum, double* correct, float* auc);",
                 "int lctr_eval_pred_weighted(lctr_ctx* ctx, int64_t n, const float* pctr, const int32_t* label, "
                 "const float* weight, float* loss_sum, double* correct, float* auc);",
                 "int lctr_train_batch_weighted_async(lctr_ctx* ctx, int64_t rows, int64_t nnz, const int64_t* row_ptr, "
                 "const uint32_t* fid, const uint16_t* field, const float* val, const int32_t* label, const float* weight, "
                 "uint64_t* ticket);"):
        assert decl in hdr, decl
