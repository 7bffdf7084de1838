"""Per-row weights without a GPU: the symbol and its Python binding, and the premises of the float64 weighted oracle of
tests/test_row_weights_gpu.py (sum_r w_r g64(row r alone))."""
import ctypes as C
import os

import numpy as np

import ref64
from conftest import ROOT
from kernel_shapes_worker import make_batch, make_params
from test_row_weights_gpu import fm_weighted64, ffm_weighted64


def test_symbol_exported_and_bound():
    from lightctr_b200 import build, capi
    assert "lctr_set_row_weights" in capi.SYMBOLS
    L = C.CDLL(build.build())
    assert hasattr(L, "lctr_set_row_weights")
    L = capi.load_library()
    assert L.lctr_set_row_weights.argtypes == [C.c_void_p, C.c_int, C.c_int64, C.c_void_p]
    hdr = open(os.path.join(ROOT, "include", "lightctr_b200.h")).read()
    assert "int lctr_set_row_weights(lctr_ctx* ctx, int slot, int64_t rows, const float* weight);" in hdr


def test_unit_weights_reproduce_the_batch_gradient():
    F, k = 500, 4
    batch = make_batch(1, F, rows=40, with_val=True)
    rp, fid, _fld, val, lab = batch
    W, V = make_params(1, F, k)
    s64, _z, p64, _sc, _c = ref64.fm_forward(rp, fid, val, W, V, k)
    want = ref64.fm_grad(rp, fid, val, lab, W, V, k, p64, s64, 1e-3)
    got = fm_weighted64(batch, W, V, k, p64, np.ones(40, np.float32), 1e-3)
    for a, b in zip(got, want):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-15)


def _duplicate(batch, counts):
    rp, fid, fld, val, lab = batch
    rows = np.repeat(np.arange(len(lab)), counts)
    idx = np.concatenate([np.arange(rp[r], rp[r + 1]) for r in rows])
    lens = np.diff(rp)[rows]
    return np.concatenate([[0], np.cumsum(lens)]).astype(np.int64), fid[idx], fld[idx], val[idx], lab[rows]


def test_integer_weights_reproduce_duplicated_rows():
    F, k, Fc = 1000, 4, 5
    batch = make_batch(2, F, rows=30, Fc=Fc, with_val=True)
    counts = np.random.default_rng(3).integers(0, 4, 30)
    W, V = make_params(2, F, k, Fc)
    p = ref64.ffm_forward(batch[0], batch[1], batch[2], batch[3], W, V, Fc, k)[1]
    got = ffm_weighted64(batch, W, V, Fc, k, p, counts.astype(np.float32), 1e-3)
    dup = _duplicate(batch, counts)
    want = ref64.ffm_grad(*dup, W, V, Fc, k, np.repeat(p, counts), 1e-3)
    for a, b in zip(got, want):
        np.testing.assert_allclose(a, b, rtol=1e-12, atol=1e-15)
