"""A train step whose working buffers cannot be allocated fails with the allocation error and leaves its buffer group
empty, with capacity 0: the next step on a smaller batch allocates again and computes what a fresh context computes.

The oversize request is sized from the device's total memory so that it exceeds the whole device; the driver refuses it
up front whatever else runs on the card, and no kernel reads a refused buffer.  What the same call allocates before it
stays well under 1 GB."""
import numpy as np
import pytest

from lightctr_b200 import capi

pytestmark = pytest.mark.gpu


def _total_memory():
    import torch
    return torch.cuda.get_device_properties(0).total_memory


def _batch(rng, rows, per_row, F, Fc=0):
    row_ptr = np.arange(rows + 1, dtype=np.int64) * per_row
    fid = rng.integers(0, F, rows * per_row).astype(np.uint32)
    field = None if not Fc else np.tile(np.arange(per_row) % Fc, rows).astype(np.uint16)
    label = rng.integers(0, 2, rows).astype(np.int32)
    return row_ptr, fid, field, label


def test_nfm_dense_layers_regrow_after_a_failed_step():
    """NFM, fp32 dense layers, deterministic = 1, one hidden layer of 65536: a step whose first layer's activations
    alone exceed the device fails; a 512-row step on another slot then matches a fresh context bit for bit."""
    F, k, H = 4096, 8, 65536
    rng = np.random.default_rng(3)
    W0 = (rng.standard_normal(F) * 0.01).astype(np.float32)
    V0 = (rng.standard_normal(F * k) * 0.05).astype(np.float32)
    layers = [((rng.standard_normal(H * k) * 0.05).astype(np.float32), (rng.standard_normal(H) * 0.01).astype(np.float32)),
              ((rng.standard_normal(H) * 0.01).astype(np.float32), np.zeros(1, np.float32))]
    x = (rng.standard_normal((512, k)) * 0.1).astype(np.float32)
    small = _batch(rng, 512, 6, F)
    big_rows = _total_memory() // (H * 4) * 5 // 4  # the first layer's activations: 1.25x the device
    big = _batch(rng, big_rows, 1, F)

    def fresh():
        ctx = capi.Context(capi.MODEL_NFM, F, k, hidden=(H,), deterministic=1)
        ctx.upload_params(W0, V0)
        for l, (w, b) in enumerate(layers):
            ctx.mlp_upload(l, w, b)
        ctx.mlp_forward(x)  # the dense buffers now hold 512 rows
        return ctx

    def state(ctx):
        W, V = ctx.download_params()
        return [W, V, *ctx.mlp_download(0, k, H), *ctx.mlp_download(1, H, 1)]

    ctx = fresh()
    row_ptr, fid, _, label = big
    ctx.upload_batch(0, row_ptr, fid, None, None, label)
    with pytest.raises(capi.LctrError, match=r"cannot allocate \d+ bytes of device memory"):
        ctx.train_step(0)
    row_ptr, fid, _, label = small
    ctx.upload_batch(1, row_ptr, fid, None, None, label)
    loss = ctx.train_step(1)[0]
    got = state(ctx)
    ctx.close()

    ref = fresh()
    ref.upload_batch(1, row_ptr, fid, None, None, label)
    ref_loss = ref.train_step(1)[0]
    want = state(ref)
    ref.close()
    assert loss == ref_loss
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


def test_grouped_ffm_tiles_regrow_after_a_failed_step():
    """Grouped FFM (deterministic = 2, field_cnt = 64, k = 8): the field-pair tile buffer takes Fc^2 * k * 4 = 128 KB per
    row; a step whose tiles exceed the device fails, and the next 512-row step matches a fresh context given the same
    parameters and optimizer state (to the tolerances of the grouped FFM tests)."""
    F, k, Fc = 20000, 8, 64
    rng = np.random.default_rng(4)
    W0 = (rng.standard_normal(F) * 0.01).astype(np.float32)
    V0 = (rng.standard_normal(F * Fc * k) * 0.05).astype(np.float32)
    small = _batch(rng, 512, 16, F, Fc)
    big_rows = _total_memory() // (Fc * Fc * k * 4) * 5 // 4
    big = _batch(rng, big_rows, 1, F, Fc)

    ctx = capi.Context(capi.MODEL_FFM, F, k, Fc, deterministic=2)
    ctx.upload_params(W0, V0)
    row_ptr, fid, field, label = small
    ctx.upload_batch(1, row_ptr, fid, field, None, label)
    ctx.train_step(1)  # the tile buffer now holds 512 rows
    W1, V1 = ctx.download_params()
    s1, s2 = ctx.download_opt_state()
    row_ptr, fid, field, label = big
    ctx.upload_batch(0, row_ptr, fid, field, None, label)
    with pytest.raises(capi.LctrError, match=r"cannot allocate \d+ bytes of device memory"):
        ctx.train_step(0)
    loss = ctx.train_step(1)[0]
    W, V = ctx.download_params()
    ctx.close()

    ref = capi.Context(capi.MODEL_FFM, F, k, Fc, deterministic=2)
    ref.upload_params(W1, V1)
    ref.upload_opt_state(s1, s2)
    row_ptr, fid, field, label = small
    ref.upload_batch(1, row_ptr, fid, field, None, label)
    ref_loss = ref.train_step(1)[0]
    Wr, Vr = ref.download_params()
    ref.close()
    assert np.allclose(loss, ref_loss, rtol=1e-6)
    assert np.max(np.abs(W - Wr)) < 1e-4 and np.max(np.abs(V - Vr)) < 1e-4
