"""tests/golden/make_ref_pins.py -- regenerates the reference side of tests/test_oracle_vs_ref.py.

Runs only where the reference sources are present: oracle/_ref/libref.so is the unmodified reference compiled in place
by oracle/Makefile (`make -C oracle ref REF=<reference checkout>`).  Every number written here is produced by the
REFERENCE on exactly the inputs the test feeds to the C oracle; the test then compares the oracle against these files on
any machine.

    python tests/golden/make_ref_pins.py <reference checkout>/data

Writes ref_pins.json (loss / accuracy bits per epoch, sha256 of parameter arrays, printed prediction lines),
ref_pins.npz (bit patterns of the sigmoid / dot / gauss vectors), train_sparse_head.csv and test_sparse_head.csv (the
first 30 rows of the reference's data/train_sparse.csv and data/test_sparse.csv: the loaders' inputs).
"""
import hashlib
import json
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
from oracle import api  # noqa: E402

HEAD_ROWS = 30


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def bits(x):
    return int(np.float32(x).view(np.uint32))


def curve(t, epochs):
    c = [t.epoch() for _ in range(epochs)]
    return dict(loss_bits=[bits(x[0]) for x in c], acc=[float(x[1]) for x in c])


def main(data):
    api.build(ref=False)
    assert api.ref_available(), "oracle/_ref/libref.so was not built (make -C oracle ref REF=<reference checkout>)"
    train, test = os.path.join(data, "train_sparse.csv"), os.path.join(data, "test_sparse.csv")
    out, arrays = {}, {}
    R = api.ref()

    # the same vectors as the test: gauss fills, dots and sigmoids of the reference
    for seed, n, k in ((1, 4096, 8), (3, 1001, 16), (9, 10, 4)):
        g = np.zeros(n, np.float32)
        R.ref_gauss_fill(seed, n, k, g)
        arrays["gauss_%d_%d_%d" % (seed, n, k)] = g.view(np.uint32)
    rng = np.random.default_rng(0)
    dots = []
    for n in (1, 3, 4, 7, 8, 9, 10, 15, 16, 17, 31, 32, 33, 64, 100, 255):
        for _ in range(20):
            x = rng.standard_normal(n).astype(np.float32)
            y = rng.standard_normal(n).astype(np.float32)
            dots.append(bits(R.ref_dot(x, y, n)))
    arrays["dot_bits"] = np.array(dots, np.uint32)
    xs = list(np.linspace(-20, 20, 4001, dtype=np.float32)) + [16.0, -16.0, 16.000002, -16.000002]
    arrays["sigmoid_bits"] = np.array([bits(R.ref_sigmoid(float(x))) for x in xs], np.uint32)

    # the loader on the head of the training file; the head of the test file for the predictors
    head, test_head = os.path.join(HERE, "train_sparse_head.csv"), os.path.join(HERE, "test_sparse_head.csv")
    for src, dst in ((train, head), (test, test_head)):
        with open(src) as f, open(dst, "w") as g:
            for _ in range(HEAD_ROWS):
                g.write(f.readline())
    t = api.RefTrainer("ffm", head, 4, field_cnt=68)
    d = t.data()
    out["loader_head"] = dict(rows=int(d.rows), nnz=int(d.nnz), feature_cnt=int(d.feature_cnt), field_cnt=int(d.field_cnt),
                              sha_row_ptr=sha(d.row_ptr), sha_fid=sha(d.fid), sha_field=sha(d.field), sha_val=sha(d.val),
                              sha_label=sha(d.label))
    t.close()

    # FM k=8, 6 epochs, then FM_Predict on the test file
    t = api.RefTrainer("fm", train, 8, seed=1, proc_cnt=1)
    W0, V0, _ = t.params()
    fm = dict(sha_W0=sha(W0), sha_V0=sha(V0), **curve(t, 6))
    W, V, S = t.params()
    fm.update(sha_W=sha(W), sha_V=sha(V), sha_sumVX=sha(S), predict_text=t.predict(test).strip(),
              predict_head_text=t.predict(test_head).strip())
    out["fm_k8_6"] = fm
    t.close()

    # FFM k=4, 68 fields, 3 epochs, then predict
    t = api.RefTrainer("ffm", train, 4, seed=1, proc_cnt=1, field_cnt=68)
    _, V0, _ = t.params()
    ffm = dict(sha_V0=sha(V0), **curve(t, 3))
    W, V, _ = t.params()
    ffm.update(sha_W=sha(W), sha_V=sha(V), predict_text=t.predict(test).strip(),
              predict_head_text=t.predict(test_head).strip())
    out["ffm_k4_3"] = ffm
    t.close()

    # NFM k=10, one hidden layer of 32, 3 epochs
    t = api.RefTrainer("nfm", train, 10, seed=1, hidden=32)
    w0, _, m0 = t.fc(0, 10, 32)
    nfm = dict(sha_fc0_w_init=sha(w0), sha_fc0_mask_init=sha(m0), **curve(t, 3))
    W, V, _ = t.params()
    w1, b1, _ = t.fc(1, 32, 1)
    nfm.update(sha_W=sha(W), sha_V=sha(V), sha_fc1_w=sha(w1), sha_fc1_b=sha(b1))
    out["nfm_k10_h32_3"] = nfm
    t.close()

    # the updaters on the test's random vectors
    rng = np.random.default_rng(5)
    n = 5000
    opt = []
    for trial in range(3):
        w = rng.standard_normal(n).astype(np.float32)
        g = (rng.standard_normal(n) * (rng.random(n) < 0.7)).astype(np.float32)
        s1 = np.abs(rng.standard_normal(n)).astype(np.float32) * (trial > 0)
        s2 = np.abs(rng.standard_normal(n)).astype(np.float32) * (trial > 0)
        rec = {}
        a = [x.copy() for x in (s1, w, g)]
        R.ref_adagrad_update(n, 1000, 0.05, a[0], a[1], a[2])
        rec["adagrad"] = [sha(x) for x in a]
        a = [x.copy() for x in (s1, w, g)]
        R.ref_rmsprop_update(n, 1000, 0.05, 0.99, a[0], a[1], a[2])
        rec["rmsprop"] = [sha(x) for x in a]
        a = [x.copy() for x in (s1, s2, w, g)]
        R.ref_adadelta_update(n, 1000, 0.8, a[0], a[1], a[2], a[3])
        rec["adadelta"] = [sha(x) for x in a]
        a = [x.copy() for x in (s1, s2, w, g)]
        R.ref_ftrl_update(n, a[0], a[1], a[2], a[3])
        rec["ftrl"] = [sha(x) for x in a]
        a = [x.copy() for x in (s1, s2, w, g)]
        R.ref_adam_update(n, 1000, 0.05, 0.8, 0.999, trial * 3, a[0], a[1], a[2], a[3])
        rec["adam"] = [sha(x) for x in a]
        opt.append(rec)
    out["optimizers"] = opt

    np.savez_compressed(os.path.join(HERE, "ref_pins.npz"), **arrays)
    with open(os.path.join(HERE, "ref_pins.json"), "w") as f:
        json.dump(out, f, indent=1)
    print("wrote ref_pins.json, ref_pins.npz, train_sparse_head.csv, test_sparse_head.csv")


if __name__ == "__main__":
    if len(sys.argv) != 2:
        sys.exit(__doc__)
    main(sys.argv[1])
