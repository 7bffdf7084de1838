"""Where a context's sparse gradient goes is decided once, from cfg (GradPath, csrc/common.cuh): compact (FM / NFM,
deterministic = 0, k in {4, 8, 16, 32}), dense (update_g + touched map + sparse apply) or feature-major (the updater inside
the backward).  This file pins the kernel launches of each path, checks that a context allocates only the gradient buffers
its path reads (lctr_device_bytes), that ranks share one IPC handle each, and that empty batches stay on the compact path."""
import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F, ROWS = 20000, 512
TWO_STATE = {1, 2, 4, 7, 8}  # FTRL, Adam, Adadelta, PS DCASGD, PS DCASGDA keep s2 beside s1


def _batch(seed=3):
    from lightctr_b200.data import CriteoSynth
    return CriteoSynth(F, seed=seed).batch(ROWS)


# name: (Context arguments, gradient path, has a predictor)
CASES = {
    "fm16_det0": (dict(model="FM", k=16, deterministic=0), "compact", True),
    "fm16_det1": (dict(model="FM", k=16, deterministic=1), "feature_major", True),
    "fm16_det2": (dict(model="FM", k=16, deterministic=2), "feature_major", True),
    "fm12_det0": (dict(model="FM", k=12, deterministic=0), "dense", True),
    "nfm16_fp32": (dict(model="NFM", k=16, deterministic=0, hidden=(32,)), "compact", False),
    "nfm16_bf16": (dict(model="NFM", k=16, deterministic=0, hidden=(64,), mlp_precision="BF16"), "compact", False),
    "nfm16_bf16_mask": (dict(model="NFM", k=16, deterministic=0, hidden=(64,), mlp_precision="BF16", mask=True), "compact",
                        False),
    "ffm4_det0": (dict(model="FFM", k=4, deterministic=0, field_cnt=39), "dense", True),
    "ffm4_det1": (dict(model="FFM", k=4, deterministic=1, field_cnt=39), "dense", True),
    "ffm4_det2": (dict(model="FFM", k=4, deterministic=2, field_cnt=39), "feature_major", True),
    "wnd": (dict(model="WND", k=8, deterministic=0, field_cnt=39, hidden=(32,)), "dense", True),
}

# NFM with mlp_precision = BF16 runs its dense chain on the wgmma kernel, or with a dropout mask on the mma.sync kernel.
# lctr_launch_count deltas of (upload, first train step, predict) on one CriteoSynth batch of ROWS rows
PINS = {
    "fm16_det0": (6, 2, 1),
    "fm16_det1": (1, 2, 1),
    "fm16_det2": (5, 3, 1),
    "fm12_det0": (1, 4, 1),
    "nfm16_fp32": (6, 16, None),
    "nfm16_bf16": (6, 5, None),
    "nfm16_bf16_mask": (6, 5, None),
    "ffm4_det0": (1, 3, 1),
    "ffm4_det1": (1, 3, 1),
    "ffm4_det2": (5, 2, 1),
    "wnd": (1, 17, 4),
}


def _ctx(capi, name, **extra):
    a, _, _ = CASES[name]
    a = dict(a)
    model = getattr(capi, "MODEL_" + a.pop("model"))
    k = a.pop("k")
    mask = a.pop("mask", False)
    if "mlp_precision" in a:
        a["mlp_precision"] = getattr(capi, "MLP_" + a["mlp_precision"])
    ctx = capi.Context(model, F, k, **a, **extra)
    if a.get("mlp_precision") == capi.MLP_BF16:  # mlp_upload writes the bf16 copies of the hidden layers
        rng = np.random.default_rng(1)
        dims = [k, *a["hidden"], 1]
        for l in range(len(dims) - 1):
            ctx.mlp_upload(l, (rng.standard_normal((dims[l + 1], dims[l])) / np.sqrt(dims[l])).astype(np.float32),
                           np.zeros(dims[l + 1], np.float32))
    if mask:  # one unit in four dropped
        ctx.mlp_set_mask(0, (np.arange(a["hidden"][0]) % 4 != 0).astype(np.float32))
    return ctx


def _upload(ctx, slot, batch):
    rp, fid, fld, lab = batch
    ctx.upload_batch(slot, rp, fid, fld if ctx.Fc else None, None, lab)


@pytest.mark.parametrize("name", sorted(CASES))
def test_launch_pins(name):
    """The launches of an upload, a train step and a predict on each path, as they were before the path was named."""
    from lightctr_b200 import capi
    ctx = _ctx(capi, name)
    batch = _batch()
    n0 = ctx.launch_count()
    _upload(ctx, 0, batch)
    n1 = ctx.launch_count()
    loss, _ = ctx.train_step(0)
    n2 = ctx.launch_count()
    assert math.isfinite(loss) and loss > 0
    got = [n1 - n0, n2 - n1, None]
    if CASES[name][2]:
        p = ctx.predict(0)
        assert np.all((p > 0) & (p < 1))
        got[2] = ctx.launch_count() - n2
    assert tuple(got) == PINS[name], (name, tuple(got))
    ctx.close()


def _shard_bytes(path, model, rowlen, two):
    """lctr_device_bytes' shard figure (include/lightctr_b200.h): W, V and s1 (+ s2), + update_g on the dense path and for
    the grouped FFM backward, + the 1-byte touched map per row on the dense path"""
    block = F * (rowlen + 1) * 4
    update_g = path == "dense" or (path == "feature_major" and model == "FFM")
    return block * (2 + two + update_g) + (F if path == "dense" else 0)


@pytest.mark.parametrize("name", sorted(CASES))
@pytest.mark.parametrize("opt", [0, 1])  # Adagrad (one state), FTRL (two)
def test_shard_bytes_follow_the_path(name, opt):
    from lightctr_b200 import capi
    ctx = _ctx(capi, name, optimizer=opt)
    a, path, _ = CASES[name]
    rowlen = a["k"] * a.get("field_cnt", 1) if a["model"] == "FFM" else a["k"]
    shard, exchange = ctx.device_bytes()
    assert shard == _shard_bytes(path, a["model"], rowlen, opt in TWO_STATE), (name, shard)
    assert exchange == 0
    ctx.close()


def test_ipc_shares_one_handle_per_rank():
    """A rank exports the handle of its arena only (one cudaIpcMemHandle_t); a blob sized for another layout is refused."""
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_FM, F, 16, world=2, rank=0, minibatch_size=ROWS)
    blob = ctx.ipc_export()
    assert len(blob) == 64
    with pytest.raises(capi.LctrError, match="bytes_per_rank"):
        ctx.ipc_import(blob * 12, 384)
    ctx.close()


def test_empty_batches_stay_on_the_compact_path():
    """One GPU, FM k=16 Adagrad, deterministic = 0: a 0-row step reports (0, 0), a step on rows without entries reports
    rows * ln 2 and 0 correct, and neither changes the parameters or the optimizer state; a normal batch then trains like
    it does on a context that never saw the empty batches."""
    from lightctr_b200 import capi
    rng = np.random.default_rng(7)
    W0 = (rng.standard_normal(F) * 0.01).astype(np.float32)
    V0 = (rng.standard_normal(F * 16) * 0.1).astype(np.float32)
    a = capi.Context(capi.MODEL_FM, F, 16, deterministic=0)
    b = capi.Context(capi.MODEL_FM, F, 16, deterministic=0)
    for c in (a, b):
        c.upload_params(W0, V0)
    before = a.download_params() + a.download_opt_state()

    a.upload_batch(1, np.zeros(1, np.int64), np.zeros(0, np.uint32), None, None, np.zeros(0, np.int32))
    n = a.launch_count()
    assert a.train_step(1) == (0.0, 0.0)
    assert a.launch_count() == n  # nothing to launch

    rows = 300
    lab = (rng.random(rows) < 0.3).astype(np.int32)
    a.upload_batch(2, np.zeros(rows + 1, np.int64), np.zeros(0, np.uint32), None, None, lab)
    loss, correct = a.train_step(2)
    assert abs(loss - rows * math.log(2.0)) <= 1e-6 * rows * math.log(2.0), loss
    assert correct == 0

    after = a.download_params() + a.download_opt_state()
    for x, y in zip(before, after):
        assert np.array_equal(x.view(np.uint32), y.view(np.uint32))

    batch = _batch(11)
    for c in (a, b):
        _upload(c, 0, batch)
    la, _ = a.train_step(0)
    lb, _ = b.train_step(0)
    assert abs(la - lb) <= 1e-6 * abs(lb), (la, lb)
    for x, y in zip(a.download_params(), b.download_params()):
        assert float(np.max(np.abs(x - y))) < 2e-5
    a.close()
    b.close()
