"""Pin the plain-C restatement (oracle/lightctr_oracle.c) bit-for-bit against the unmodified reference.  The reference
side was recorded by running the reference compiled in place (oracle/_ref/libref.so) on exactly these inputs
(tests/golden/make_ref_pins.py -> tests/golden/ref_pins.json, ref_pins.npz, train_sparse_head.csv, test_sparse_head.csv);
the training data is the reference's own data/train_sparse.csv and test_sparse.csv as its parser reads them
(train_sparse_csr.npz, test_sparse_csr.npz).  CPU-only."""
import hashlib
import json
import os

import numpy as np
import pytest

from golden_util import GOLDEN, load_csr, write_libffm

HEAD = os.path.join(GOLDEN, "train_sparse_head.csv")
TEST_HEAD = os.path.join(GOLDEN, "test_sparse_head.csv")


@pytest.fixture(scope="module")
def pins():
    with open(os.path.join(GOLDEN, "ref_pins.json")) as f:
        return json.load(f)


@pytest.fixture(scope="module")
def pin_arrays():
    return np.load(os.path.join(GOLDEN, "ref_pins.npz"))


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def bits(x):
    return int(np.float32(x).view(np.uint32))


def test_rand_stream_matches_glibc(oracle_api):
    import ctypes
    libc = ctypes.CDLL("libc.so.6")
    L = oracle_api.lib()
    for seed in (1, 7, 12345, 0):
        libc.srand(seed)
        L.orc_srand(seed)
        a = [libc.rand() for _ in range(1000)]
        b = [L.orc_rand() for _ in range(1000)]
        assert a == b


def test_gauss_init_bit_exact(oracle_api, pin_arrays):
    for seed, n, k in ((1, 4096, 8), (3, 1001, 16), (9, 10, 4)):
        ref = pin_arrays["gauss_%d_%d_%d" % (seed, n, k)]
        L = oracle_api.lib()
        L.orc_srand(seed)
        L.orc_gauss_reset()
        mine = np.zeros(n, np.float32)
        L.orc_init_V(mine, n, k)
        assert np.array_equal(ref, mine.view(np.uint32))


def test_dot_and_sigmoid_bit_exact(oracle_api, pin_arrays):
    rng = np.random.default_rng(0)
    L = oracle_api.lib()
    dots = []
    for n in (1, 3, 4, 7, 8, 9, 10, 15, 16, 17, 31, 32, 33, 64, 100, 255):
        for _ in range(20):
            x = rng.standard_normal(n).astype(np.float32)
            y = rng.standard_normal(n).astype(np.float32)
            dots.append(bits(L.orc_dot(x, y, n)))
    assert np.array_equal(np.array(dots, np.uint32), pin_arrays["dot_bits"])
    xs = list(np.linspace(-20, 20, 4001, dtype=np.float32)) + [16.0, -16.0, 16.000002, -16.000002]
    sig = np.array([bits(L.orc_sigmoid(float(x))) for x in xs], np.uint32)
    assert np.array_equal(sig, pin_arrays["sigmoid_bits"])


def test_loader_bit_exact(oracle_api, pins, tmp_path):
    # the reference's own bytes (head of the training file) against the reference parser's arrays
    p = pins["loader_head"]
    d = oracle_api.load(HEAD, field_cnt=68)
    assert (d.rows, d.nnz, d.feature_cnt, d.field_cnt) == (p["rows"], p["nnz"], p["feature_cnt"], p["field_cnt"])
    for a, key in ((d.row_ptr, "sha_row_ptr"), (d.fid, "sha_fid"), (d.field, "sha_field"), (d.val, "sha_val"),
                   (d.label[:d.rows], "sha_label")):
        assert sha(a) == p[key], key
    # the whole training file, written back out from the reference parser's arrays
    ref = load_csr("train_sparse_csr.npz", field_cnt=68)
    path = str(tmp_path / "train.txt")
    write_libffm(ref, path)
    d = oracle_api.load(path, field_cnt=68)
    assert (d.rows, d.nnz, d.feature_cnt, d.field_cnt) == (1000, 281975, 233789, 68)
    for a, b in ((d.row_ptr, ref.row_ptr), (d.fid, ref.fid), (d.field, ref.field), (d.val, ref.val),
                 (d.label[:d.rows], ref.label[:ref.rows])):
        assert np.array_equal(a, b)


def _predict_head(oracle_api, p, ds, Fc, k, o, sumVX, is_ffm):
    """load_test on the reference's own test-file bytes, then the predictor against the reference's printed line."""
    head = oracle_api.load_test(TEST_HEAD, ds.feature_cnt)
    full = load_csr("test_sparse_csr.npz")
    assert head.rows == 30
    assert np.array_equal(head.row_ptr, full.row_ptr[:31]) and np.array_equal(head.fid, full.fid[:head.nnz])
    assert np.array_equal(head.label[:30], full.label[:30])
    _, loss, _, auc = oracle_api.predict(head, Fc, k, o.W, o.V, sumVX, is_ffm)
    ref_loss, _, ref_auc = _predict_line(p["predict_head_text"])
    assert ref_loss in (float("%.6g" % loss), float("%.5g" % loss))
    assert float("%.4f" % auc) == ref_auc


def _curve(o, p, exact_acc=True):
    for e, (lb, ar) in enumerate(zip(p["loss_bits"], p["acc"])):
        lo, ao = o.epoch()
        assert bits(lo) == lb, (e, lo)
        if exact_acc:
            assert ao == ar, (e, ao, ar)
        else:
            assert ao == pytest.approx(ar, abs=1e-7)


def _predict_line(text):
    return (float(text.split("likelihood = ")[1].split()[0]), float(text.split("correct = ")[1].split()[0]),
            float(text.split("auc = ")[1].split()[0]))


def test_fm_training_bit_exact(oracle_api, pins):
    p = pins["fm_k8_6"]
    k = 8
    ds = load_csr("train_sparse_csr.npz")
    Wi, Vi = oracle_api.init_params(1, ds.feature_cnt, k)
    assert sha(Vi) == p["sha_V0"] and sha(Wi) == p["sha_W0"]
    o = oracle_api.FMOracle(ds, k, Wi, Vi)
    _curve(o, p)
    assert sha(o.W) == p["sha_W"] and sha(o.V) == p["sha_V"] and sha(o.sumVX) == p["sha_sumVX"]
    # FM_Predict with its quirks (predict/fm_predict.cpp)
    test = load_csr("test_sparse_csr.npz")
    pctr, loss, correct, auc = oracle_api.predict(test, 0, k, o.W, o.V, o.sumVX, False)
    assert test.rows == 200
    ref_loss, ref_acc, ref_auc = _predict_line(p["predict_text"])
    assert ref_loss in (float("%.6g" % loss), float("%.5g" % loss))
    assert float("%.5g" % (np.float32(correct) / np.float32(test.rows))) == pytest.approx(ref_acc, rel=1e-6)
    assert float("%.4f" % auc) == ref_auc
    _predict_head(oracle_api, p, ds, 0, k, o, o.sumVX, False)


def test_ffm_training_bit_exact(oracle_api, pins):
    p = pins["ffm_k4_3"]
    k, Fc = 4, 68
    ds = load_csr("train_sparse_csr.npz", field_cnt=Fc)
    Wi, Vi = oracle_api.init_params(1, ds.feature_cnt, k, Fc)
    assert sha(Vi) == p["sha_V0"]
    o = oracle_api.FFMOracle(ds, k, Wi, Vi)
    _curve(o, p)
    assert sha(o.W) == p["sha_W"] and sha(o.V) == p["sha_V"]
    test = load_csr("test_sparse_csr.npz")
    pctr, loss, correct, auc = oracle_api.predict(test, Fc, k, o.W, o.V, None, True)
    # cout keeps setprecision(5) from an earlier Predict() in this process (fm_predict.cpp:73-74)
    ref_loss, _, ref_auc = _predict_line(p["predict_text"])
    assert ref_loss in (float("%.6g" % loss), float("%.5g" % loss))
    assert float("%.4f" % auc) == ref_auc
    _predict_head(oracle_api, p, ds, Fc, k, o, None, True)


def test_nfm_training_bit_exact(oracle_api, pins):
    p = pins["nfm_k10_h32_3"]
    k, H = 10, 32
    ds = load_csr("train_sparse_csr.npz")
    o = oracle_api.NFMOracle(ds, k, H, seed=1)
    assert sha(o.mlp.arrays("weight", 0)) == p["sha_fc0_w_init"]
    assert sha(o.mlp.arrays("mask", 0)) == p["sha_fc0_mask_init"]
    _curve(o, p, exact_acc=False)
    assert sha(o.W) == p["sha_W"] and sha(o.V) == p["sha_V"]
    assert sha(o.mlp.arrays("weight", 1)) == p["sha_fc1_w"]
    assert sha(o.mlp.arrays("bias", 1)) == p["sha_fc1_b"]


def test_optimizer_units_bit_exact(oracle_api, pins):
    rng = np.random.default_rng(5)
    L = oracle_api.lib()
    n = 5000
    import ctypes as C
    for trial in range(3):
        ref = pins["optimizers"][trial]
        w = rng.standard_normal(n).astype(np.float32)
        g = (rng.standard_normal(n) * (rng.random(n) < 0.7)).astype(np.float32)
        s1 = np.abs(rng.standard_normal(n)).astype(np.float32) * (trial > 0)
        s2 = np.abs(rng.standard_normal(n)).astype(np.float32) * (trial > 0)
        b = [x.copy() for x in (s1, w, g)]
        L.orc_adagrad(n, b[1], b[2], b[0], 1000, 0.05)
        assert [sha(x) for x in b] == ref["adagrad"], trial
        b = [x.copy() for x in (s1, w, g)]
        L.orc_rmsprop(n, b[1], b[2], b[0], 1000, 0.05, 0.99)
        assert [sha(x) for x in b] == ref["rmsprop"], trial
        b = [x.copy() for x in (s1, s2, w, g)]
        L.orc_adadelta(n, b[2], b[3], b[0], b[1], 1000, 0.8)
        assert [sha(x) for x in b] == ref["adadelta"], trial
        b = [x.copy() for x in (s1, s2, w, g)]
        L.orc_ftrl(n, b[2], b[3], b[0], b[1], 0)
        assert [sha(x) for x in b] == ref["ftrl"], trial
        b = [x.copy() for x in (s1, s2, w, g)]
        it = C.c_size_t(trial * 3)
        L.orc_adam(n, b[2], b[3], b[0], b[1], C.byref(it), 1000, 0.05, 0.8, 0.999)
        assert [sha(x) for x in b] == ref["adam"], trial
