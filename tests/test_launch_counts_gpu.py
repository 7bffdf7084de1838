"""Kernel launches of the calls outside a train step, counted by lctr_launch_count: the metrics, the stand-alone dense
chain, the streamed pipeline on and off its captured graphs, a checkpoint load into a dense context and the weight
upload of a bf16 context.  The train step's own pins are in test_grad_path_gpu.py, the keyed calls' in
test_keyed_launches_gpu.py."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

F, ROWS = 20000, 512


def _batch(seed):
    from lightctr_b200.data import CriteoSynth
    return CriteoSynth(F, seed=seed).batch(ROWS)


def _delta(ctx, fn):
    n = ctx.launch_count()
    fn()
    return ctx.launch_count() - n


def eval_counts():
    """(predict, eval) on a trained FM context"""
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_FM, F, 16)
    rp, fid, _, lab = _batch(3)
    ctx.upload_batch(0, rp, fid, None, None, lab)
    ctx.train_step(0)
    got = (_delta(ctx, lambda: ctx.predict(0)), _delta(ctx, lambda: ctx.eval_metrics(0)))
    ctx.close()
    return got


def mlp_operator_counts():
    """(forward, backward, apply) of lctr_mlp_* on an fp32 chain 12 -> 20 -> 8 -> 1"""
    from lightctr_b200 import capi
    dims, rows = [12, 20, 8, 1], 48
    ctx = capi.Context(capi.MODEL_NFM, 1, dims[0], hidden=tuple(dims[1:-1]), minibatch_size=rows)
    rng = np.random.default_rng(0)
    x = rng.standard_normal((rows, dims[0])).astype(np.float32)
    dout = rng.standard_normal(rows).astype(np.float32)
    got = (_delta(ctx, lambda: ctx.mlp_forward(x)), _delta(ctx, lambda: ctx.mlp_backward(dout, dims[0])),
           _delta(ctx, lambda: ctx.mlp_apply(rows)))
    ctx.close()
    return got


# name: (k, deterministic, on the captured graphs)
ASYNC = {
    "fm16_det0": (16, 0, True),
    "fm16_det2": (16, 2, True),
    "fm12_det0": (12, 0, False),
}


def async_counts(name):
    """launches of each of four lctr_train_batch_async calls (the first captures the graphs of its pipeline slot)"""
    from lightctr_b200 import capi
    k, det, _ = ASYNC[name]
    ctx = capi.Context(capi.MODEL_FM, F, k, deterministic=det)
    batches = [_batch(20 + i) for i in range(4)]
    got, tickets = [], []
    for rp, fid, _, lab in batches:
        n = ctx.launch_count()
        tickets.append(ctx.train_batch_async(rp, fid, None, None, lab))
        got.append(ctx.launch_count() - n)
        if len(tickets) == capi.PIPE_DEPTH:
            ctx.wait(tickets.pop(0))
    for t in tickets:
        ctx.wait(t)
    ctx.close()
    return tuple(got)


def checkpoint_shards_counts(tmp):
    """lctr_load_checkpoint_shards of a one-GPU FM and FFM file into rank 0 of two (the reshard kernels)"""
    import os
    from lightctr_b200 import capi
    got = []
    for model, k, fc in ((capi.MODEL_FM, 16, 0), (capi.MODEL_FFM, 4, 39)):
        a = capi.Context(model, F, k, fc)
        rp, fid, fld, lab = _batch(3)
        a.upload_batch(0, rp, fid, fld if fc else None, None, lab)
        a.train_step(0)
        path = os.path.join(tmp, "m%d.ckpt" % model)
        a.save_checkpoint(path)
        a.close()
        b = capi.Context(model, F, k, fc, world=2, rank=0, minibatch_size=ROWS)
        got.append(_delta(b, lambda: b.load_checkpoint_shards([path])))
        b.close()
    return tuple(got)


def bf16_upload_counts():
    """lctr_mlp_upload of each layer of a bf16 NFM chain 16 -> 64 -> 1: the hidden layer refreshes its bf16 copies"""
    from lightctr_b200 import capi
    dims = [16, 64, 1]
    ctx = capi.Context(capi.MODEL_NFM, F, dims[0], hidden=(dims[1],), mlp_precision=capi.MLP_BF16)
    rng = np.random.default_rng(1)
    got = tuple(_delta(ctx, lambda: ctx.mlp_upload(l, rng.standard_normal((dims[l + 1], dims[l])).astype(np.float32),
                                                   np.zeros(dims[l + 1], np.float32))) for l in range(len(dims) - 1))
    ctx.close()
    return got


def test_eval_launches():
    assert eval_counts() == (1, 5)


def test_mlp_operator_launches():
    assert mlp_operator_counts() == (3, 9, 6)


# graph path: each pipeline slot captures its two graphs on first use (8 kernels) and replays them (8 more)
ASYNC_PINS = {
    "fm16_det0": (16, 16, 16, 8),
    "fm16_det2": (16, 16, 16, 8),
    "fm12_det0": (5, 5, 5, 5),
}


@pytest.mark.parametrize("name", sorted(ASYNC))
def test_train_batch_async_launches(name):
    assert async_counts(name) == ASYNC_PINS[name]


def test_load_checkpoint_shards_launches(tmp_path):
    assert checkpoint_shards_counts(str(tmp_path)) == (4, 4)  # W, V, s1W, s1V: one chunk each


def test_bf16_mlp_upload_launches():
    """one to_bf16 launch for the hidden layer, none for the fp32 output layer"""
    assert bf16_upload_counts() == (1, 0)
