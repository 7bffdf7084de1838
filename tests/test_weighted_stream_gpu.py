"""Weighted batches through the streamed pipeline (lctr_train_batch_weighted_async / lctr_wait) against a twin context
that trains the same batches with lctr_upload_batch + lctr_set_row_weights + lctr_train_step: bit for bit on batches whose
gradients are exact in fp32 (tests/exact_batch.py, weights 0 and 1), within 1e-6 on random batches under plain SGD (3e-5
for the bf16 dense layers), and the lctr_wait statistics equal to the twin's.  FM runs on the captured-graph path (compact, device-grouped) and on the dense path; FFM,
NFM (fp32 and bf16 dense layers) and Wide&Deep stream on the launch path.  Two ranks through tests/multirank.py:
dist.eval_global with weights, and a weighted two-rank stream against a world-1 context on the joined batch."""
import numpy as np
import pytest

import exact_batch as eb
import multirank as mr

pytestmark = pytest.mark.gpu

PIPE = 3  # LCTR_PIPE_DEPTH
F, ROWS, STEPS = 20000, 512, 2 * PIPE + 1

# name: (model, k, deterministic, mlp precision or None)
CONFIGS = {
    "fm-compact": ("fm", 16, 0, None),
    "fm-grouped": ("fm", 16, 2, None),
    "fm-dense": ("fm", 12, 0, None),
    "ffm": ("ffm", 4, 0, None),
    "nfm-fp32": ("nfm", 16, 0, "fp32"),
    "nfm-bf16": ("nfm", 16, 0, "bf16"),
    "wnd": ("wnd", 8, 0, None),
}


def _ctx(name):
    from lightctr_b200 import capi
    model, k, det, prec = CONFIGS[name]
    # plain SGD: the RED-scatter paths sum in arbitrary order, and an adaptive rule would magnify those last bits where a
    # coordinate's gradient nearly cancels
    kw = {"deterministic": det, "optimizer": capi.OPT_PS_SGD}
    if prec:
        kw["mlp_precision"] = capi.MLP_BF16 if prec == "bf16" else capi.MLP_FP32
    ctx = mr.make_context(model, F, k, 0, 1, minibatch_size=ROWS, max_nnz=ROWS * 400, **kw)
    ctx.upload_params(*mr.make_params(F, k, model))
    for l, (w, b) in enumerate(mr.dense_layers(model, k)):
        ctx.mlp_upload(l, w, b)
    return ctx


def _weights(i, rows, kind="random"):
    rng = np.random.default_rng(40 + i)
    if kind == "ones":
        return np.ones(rows, np.float32)
    if kind == "binary":
        return (rng.random(rows) < 0.7).astype(np.float32)
    w = (rng.random(rows) * 3).astype(np.float32)
    w[::9] = 0.0
    return w


def _params(ctx, name):
    model, k = CONFIGS[name][:2]
    out = list(ctx.download_params())
    dims = mr.layer_dims(model, k)
    for l in range(len(dims) - 1):
        out += list(ctx.mlp_download(l, dims[l], dims[l + 1]))
    return out


def _stream(ctx, batches, ws, fc):
    """every batch through the pipeline (None weights: the unweighted call), at most PIPE in flight; the wait statistics"""
    tickets, stats = [], []
    for i, (b, w) in enumerate(zip(batches, ws)):
        if i >= PIPE:
            stats.append(ctx.wait(tickets[i - PIPE]))
        rp, fid, fld, lab = b
        tickets.append(ctx.train_batch_async(rp, fid, fld if fc else None, None, lab, weight=w))
    stats += [ctx.wait(t) for t in tickets[len(stats):]]
    return stats


def _twin(ctx, model, batches, ws):
    stats = []
    for b, w in zip(batches, ws):
        mr.upload(ctx, model, 0, b)
        if w is not None:
            ctx.set_row_weights(0, w)
        stats.append(ctx.train_step(0))
    return stats


def _close(what, got, want, tol):
    for i, (a, b) in enumerate(zip(got, want)):
        np.testing.assert_allclose(a, b, rtol=tol, atol=tol, err_msg="%s, array %d" % (what, i))


def _same(what, got, want):
    for i, (a, b) in enumerate(zip(got, want)):
        a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
        bad = np.flatnonzero(a.view(np.uint32) != b.view(np.uint32))
        assert len(bad) == 0, "%s, array %d: %d differ, first at %d: %r vs %r" % (what, i, len(bad), bad[0], a[bad[0]], b[bad[0]])


def _stats_close(got, want, tol=1e-6):
    for (gl, ga), (wl, wa) in zip(got, want):
        assert abs(gl - wl) <= tol * abs(wl), (gl, wl)
        assert abs(ga - wa) <= tol * abs(wa) + 1e-3, (ga, wa)


def _run_pair(name, ws, batches=None):
    model = CONFIGS[name][0]
    batches = batches or mr.train_batches(F, ROWS, len(ws), 0)
    a, b = _ctx(name), _ctx(name)
    got = _stream(a, batches, ws, mr.field_cnt(model))
    want = _twin(b, model, batches, ws)
    pa, pb = _params(a, name), _params(b, name)
    a.close()
    b.close()
    return got, want, pa, pb


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_weighted_stream_equals_twin(name):
    ws = [_weights(i, ROWS) for i in range(STEPS)]
    got, want, pa, pb = _run_pair(name, ws)
    _stats_close(got, want, 1e-5)  # the pCTR of both follow parameters that differ in their last bits
    # bf16 dense layers: a last-bit difference of an activation can move it across a bf16 rounding boundary
    _close(name, pa, pb, 3e-5 if CONFIGS[name][3] == "bf16" else 1e-6)


@pytest.mark.parametrize("name", ["fm-compact", "fm-grouped", "fm-dense"])
def test_alternating_weighted_and_unweighted(name):
    """each pipeline slot changes kind from one use to the next: the graph path recaptures, the launch path relabels"""
    ws = [_weights(i, ROWS) if i % 2 else None for i in range(STEPS + 2)]
    got, want, pa, pb = _run_pair(name, ws)
    _stats_close(got, want, 1e-5)
    if CONFIGS[name][2] == 2:
        _same(name, pa, pb)
    else:
        _close(name, pa, pb, 1e-6)


# exact batches (tests/exact_batch.py): FM and FFM, weights 0 and 1, one updater rule
EXACT = {"fm-compact": (16, 0, 0), "fm-grouped": (16, 0, 2), "fm-dense": (12, 0, 0), "ffm": (4, 3, 0)}


def _exact_ctx(k, Fc, det, l2):
    from lightctr_b200 import capi
    h = eb.HYPER
    return capi.Context(capi.MODEL_FFM if Fc else capi.MODEL_FM, 3000, k, Fc, optimizer=eb.capi_opt("adagrad"),
                        lr=h["lr"], l2=l2, minibatch_size=0, deterministic=det)


def _exact_params(batches, seed):
    """W0 / V0 as tests/test_updaters_gpu.py sets them up: each batch has ids of its own, so its gradient stays exact"""
    W0, V0 = eb.make_params(batches[0], seed)
    b0 = batches[0]
    for b in batches:
        V0.reshape(3000, b0.rowlen)[b.single_only[::2]] = 0
    return W0, V0


@pytest.mark.parametrize("name", sorted(EXACT))
def test_weighted_stream_bit_for_bit_on_exact_batches(name):
    k, Fc, det = EXACT[name]
    n, span = STEPS, 3000 // STEPS
    batches = [eb.make_batch(90 + i, 3000, k, Fc, scale=eb.SCALE["adagrad"], rows=280, id_base=i * span, id_span=span)
               for i in range(n)]
    W0, V0 = _exact_params(batches, 90)
    ws = [_weights(i, batches[i].rows, "binary") for i in range(n)]
    a, b = _exact_ctx(k, Fc, det, batches[0].l2), _exact_ctx(k, Fc, det, batches[0].l2)
    for c in (a, b):
        c.upload_params(W0, V0)
    tickets, got = [], []
    for i, (bt, w) in enumerate(zip(batches, ws)):
        if i >= PIPE:
            got.append(a.wait(tickets[i - PIPE]))
        tickets.append(a.train_batch_async(bt.rp, bt.fid, bt.fld if Fc else None, bt.val, bt.lab, weight=w))
    got += [a.wait(t) for t in tickets[len(got):]]
    want = []
    for bt, w in zip(batches, ws):
        b.upload_batch(0, bt.rp, bt.fid, bt.fld if Fc else None, bt.val, bt.lab)
        b.set_row_weights(0, w)
        want.append(b.train_step(0))
    _same(name, a.download_params(), b.download_params())
    _stats_close(got, want)
    a.close()
    b.close()


def test_unit_weights_bit_for_bit_with_deterministic_2():
    """w = 1 streams bit for bit as the unweighted stream (FM, device grouping, on the captured graphs)"""
    batches = mr.train_batches(F, ROWS, STEPS, 0)
    a, b = _ctx("fm-grouped"), _ctx("fm-grouped")
    sa = _stream(a, batches, [np.ones(ROWS, np.float32)] * STEPS, 0)
    sb = _stream(b, batches, [None] * STEPS, 0)
    _same("fm-grouped", a.download_params(), b.download_params())
    _stats_close(sa, sb)  # (the weighted statistics sum in another order than the forward's)
    a.close()
    b.close()


def _null_weight_call(ctx, bt):
    import ctypes as C
    t = C.c_uint64()
    rc = ctx.L.lctr_train_batch_weighted_async(ctx.h, bt.rows, len(bt.fid), bt.rp.ctypes.data, bt.fid.ctypes.data, None,
                                               bt.val.ctypes.data, bt.lab.ctypes.data, None, C.byref(t))
    assert rc == 0
    return t.value


@pytest.mark.parametrize("name", ["fm-grouped", "fm-dense"])
def test_null_weight_is_the_unweighted_call(name):
    """weight = NULL: the same launches per call and the same parameters as lctr_train_batch_async (exact batches)"""
    k, Fc, det = EXACT[name]
    span = 3000 // 5
    batches = [eb.make_batch(70 + i, 3000, k, 0, scale=eb.SCALE["adagrad"], rows=280, id_base=i * span, id_span=span)
               for i in range(5)]
    W0, V0 = _exact_params(batches, 70)
    res = []
    for weighted_entry in (False, True):
        c = _exact_ctx(k, 0, det, batches[0].l2)
        c.upload_params(W0, V0)
        counts, tickets = [], []
        for bt in batches:
            n = c.launch_count()
            tickets.append(_null_weight_call(c, bt) if weighted_entry else
                           c.train_batch_async(bt.rp, bt.fid, None, bt.val, bt.lab))
            counts.append(c.launch_count() - n)
            if len(tickets) == PIPE:
                c.wait(tickets.pop(0))
        for t in tickets:
            c.wait(t)
        res.append((counts, c.download_params()))
        c.close()
    assert res[0][0] == res[1][0]
    _same(name, res[0][1], res[1][1])


def test_refused_weights_issue_no_ticket():
    from lightctr_b200 import capi
    ctx = _ctx("fm-compact")
    batches = mr.train_batches(F, ROWS, 3, 0)
    w = _weights(0, ROWS)
    t0 = ctx.train_batch_async(*batches[0][:2], None, None, batches[0][3], weight=w)
    for bad in (np.nan, -0.5, np.inf):
        wb = w.copy()
        wb[100] = bad
        n = ctx.launch_count()
        with pytest.raises(capi.LctrError, match="not a finite value"):
            ctx.train_batch_async(*batches[1][:2], None, None, batches[1][3], weight=wb)
        assert ctx.launch_count() == n
    t1 = ctx.train_batch_async(*batches[1][:2], None, None, batches[1][3], weight=w)
    assert t1 == t0 + 1
    ctx.wait(t0)
    ctx.wait(t1)
    ctx.close()


# graph path: a weighted step graph has one node more (the weighted statistics): capture 9 + replay 9, then 9; the launch
# path launches the statistics once per step
WEIGHTED_PINS = {"fm-compact": (18, 18, 18, 9), "fm-grouped": (18, 18, 18, 9), "fm-dense": (6, 6, 6, 6)}


@pytest.mark.parametrize("name", sorted(WEIGHTED_PINS))
def test_weighted_stream_launches(name):
    from lightctr_b200 import capi
    model, k, det, _ = CONFIGS[name]
    ctx = capi.Context(capi.MODEL_FM, F, k, deterministic=det)
    got, tickets = [], []
    for i, (rp, fid, _f, lab) in enumerate(mr.train_batches(F, ROWS, 4, 0)):
        w = _weights(i, ROWS)
        n = ctx.launch_count()
        tickets.append((ctx.train_batch_async(rp, fid, None, None, lab, weight=w), w))
        got.append(ctx.launch_count() - n)
        if len(tickets) == PIPE:
            ctx.wait(tickets.pop(0)[0])
    for t, _w in tickets:
        ctx.wait(t)
    ctx.close()
    assert tuple(got) == WEIGHTED_PINS[name]


# ------------------------------------------------------------------------------------------------------------------------
# two ranks on one GPU (tests/dist_weighted_stream_worker.py)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shares", ["300,0", "257,1000", "0,64"])
def test_two_ranks_weighted_eval_global(tmp_path, shares):
    mr.launch("dist_weighted_stream_worker.py", tmp_path, ["--mode", "metrics", "--test-rows-per-rank", shares])
    parts, res = mr.load(tmp_path), mr.load_json(tmp_path)
    assert res[0]["metrics"] == res[1]["metrics"]
    for o in res:
        assert o["mismatch"] is not None and "rank(s) [1]" in o["mismatch"], o["mismatch"]
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_FM, 100, 4)
    cat = [np.concatenate([p[key] for p in parts]) for key in ("pctr", "label", "weight")]
    want = ctx.eval_pred(*cat)
    ctx.close()
    got = res[0]["metrics"]
    assert np.float32(got[0]).view(np.uint32) == np.float32(want[0]).view(np.uint32), (got, want)
    assert got[1] == want[1], (got, want)
    assert np.float32(got[2]).view(np.uint32) == np.float32(want[2]).view(np.uint32), (got, want)


@pytest.mark.parametrize("model,k", [("fm", 16), ("ffm", 4), ("nfm", 16)])
def test_two_ranks_weighted_stream_equal_world1(tmp_path, model, k):
    """parameters and the ranks' summed wait statistics equal a world-1 context trained on multirank.global_batch with the
    concatenated weights, to the two-rank tolerance (the sparse scatter sums in arbitrary order)"""
    import dist_weighted_stream_worker as wk
    from lightctr_b200 import dist as ldist
    rows = 256
    mr.launch("dist_weighted_stream_worker.py", tmp_path, ["--mode", "stream", "--model", model, "--k", str(k),
                                                           "--rows", str(rows)])
    parts, res = mr.load(tmp_path), mr.load_json(tmp_path)
    ctx = mr.make_context(model, 20000, k, 0, 1, minibatch_size=2 * rows, max_nnz=rows * 400)
    ctx.upload_params(*mr.make_params(20000, k, model))
    for l, (w, b) in enumerate(mr.dense_layers(model, k)):
        ctx.mlp_upload(l, w, b)
    per_rank = [mr.train_batches(20000, rows, wk.STEPS, r) for r in range(2)]
    for i in range(wk.STEPS):
        mr.upload(ctx, model, 0, mr.global_batch([per_rank[r][i] for r in range(2)]))
        ctx.set_row_weights(0, np.concatenate([wk.weights(r, i, len(per_rank[r][i][3])) for r in range(2)]))
        loss, acc = ctx.train_step(0)
        got_l = sum(res[r]["loss"][i] for r in range(2))
        got_a = sum(res[r]["acc"][i] for r in range(2))
        assert abs(got_l - loss) <= 1e-5 * abs(loss), (i, got_l, loss)
        assert abs(got_a - acc) <= 1e-5 * abs(acc) + 1e-3, (i, got_a, acc)
    W, V = ctx.download_params()
    dims = mr.layer_dims(model, k)
    dense = [ctx.mlp_download(l, dims[l], dims[l + 1]) for l in range(len(dims) - 1)]
    ctx.close()
    assert np.max(np.abs(ldist.merge_shards([p["W"] for p in parts], 2, 20000) - W)) < 1e-5
    assert np.max(np.abs(ldist.merge_shards([p["V"] for p in parts], 2, 20000) - V)) < 1e-5
    for l, (w, b) in enumerate(dense):
        for p in parts:
            assert np.max(np.abs(p["mlp_w%d" % l] - w)) < 1e-5 and np.max(np.abs(p["mlp_b%d" % l] - b)) < 1e-5
