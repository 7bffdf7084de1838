"""Every Wide&Deep path (LCTR_MODEL_WND: csrc/wnd.cu and the fp32 dense layers of csrc/mlp.cu) against tests/ref64.py.
Each test id names the kernels and the shape it reaches.

The probe of tests/test_gradients_gpu.py: OPT_PS_SGD with lr = minibatch_size = 1, so g = w0 - w1 for the wide weights W
and the tensors E.  Per step:
- the step's pCTR against ref64.wnd_forward + ref64.nfm_head;
- gW against ref64.wnd_grad at the kernel's own pCTR, gE against the scatter of ref64's dz by first-entry fid, both
  within ref64.probe_excess;
- W moved on exactly the ids of the stepped rows, E on exactly the fids that are the first entry of some field of a
  stepped row (rows of weight 0 move nothing);
- on the first step of a context (LCTR_MLP_SKIP_UPDATE=1 leaves the dense layers and their gradient buffer as the step
  wrote them), every layer's dW / db against nfm_head's, within 1e-5 of their condition figures.

wnd_forward_kernel walks a row 32 entries at a time: a field's first entry is the lowest lane of __match_any_sync inside a
chunk whose bit is not yet set in the warp's `seen` bitmap of ceil(Fc / 32) words, so the batches hold rows of 31, 32,
33, 64, 65 and 300 entries with a field first at lane 31 and again in the next chunk, and a field only past entry 31."""
import numpy as np
import pytest

import ref64
from kernel_shapes_worker import make_params
from test_gradients_gpu import _check_grad, _check_moved, _check_pctr, _rows, _step, _unit_sgd_context

pytestmark = pytest.mark.gpu

F = 5000
SPECIAL = (0, 1, 31, 32, 33, 64, 65, 300)


def wnd_batch(seed, Fc, rows, with_val):
    """rows of 0, 1, 31, 32, 33, 64, 65 and 300 entries spread over the slot, the others 2..40; ids 0..2 shared by most
    rows, the rest distinct within a row; fields random (unsorted, repeated, absent).  With Fc >= 2 the fid of entry 0 is
    also entry 1, the first entry of a second field; every row of 4 or more repeats a fid; in every row of more than 32
    entries (Fc >= 4) field A is first at entry 31 (lane 31 of chunk 0), and again at entry 33 when there is one, and field
    B lies only in the last chunk.  Returns rp, fid, fld (uint16), val (None when absent), lab."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(2, 41, rows)
    lens[np.arange(len(SPECIAL)) * (rows // len(SPECIAL)) + 3] = SPECIAL
    fids, flds = [], []
    for r, n in enumerate(lens):
        ids = rng.choice(np.arange(3, F), n, replace=False)
        fl = rng.integers(0, Fc, n)
        if n >= 3:
            ids[int(rng.integers(2, n))] = r % 3
        if n >= 2 and Fc >= 2:
            ids[1], fl[1] = ids[0], (fl[0] + 1) % Fc
        if n >= 4:
            ids[n - 2] = ids[2]
        if n > 32 and Fc >= 4:
            a, b = (fl[0] + 2) % Fc, (fl[0] + 3) % Fc
            last = (n - 1) // 32 * 32
            mid = fl[2:last]
            mid[(mid == a) | (mid == b)] = fl[0]
            fl[31], fl[n - 1] = a, b
            if n > 34:
                fl[33] = a
        fids.append(ids)
        flds.append(fl)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fid = np.concatenate(fids).astype(np.uint32)
    fld = np.concatenate(flds).astype(np.uint16)
    val = (0.25 + 1.5 * rng.random(len(fid))).astype(np.float32) if with_val else None
    lab = (rng.random(rows) < 0.4).astype(np.int32)
    return rp, fid, fld, val, lab


def wnd_layers(seed, dims):
    rng = np.random.default_rng(seed + 7)
    return [(((rng.random((dims[i + 1], dims[i])) - 0.5) * (3 / np.sqrt(dims[i]))).astype(np.float32),
             (rng.standard_normal(dims[i + 1]) * 0.1).astype(np.float32)) for i in range(len(dims) - 1)]


def check_wnd(sub, W0, E0, W1, E1, pred, Fc, d, layers, act, l2, weights=None, dense=None):
    """the probe's checks on the rows `sub` of one step; dense: the step's [(dW, db)] per layer, or None"""
    rp, fid, fld, val, lab = sub
    z, first, wide, z_c, w_c = ref64.wnd_forward(rp, fid, fld, val, W0, E0, Fc, d)
    p64, dz, dz_c, logit_c, grads = ref64.nfm_head(z, wide, layers, act, None, lab, z_c, w_c, weights=weights,
                                                   grads=True)
    _check_pctr(pred, p64, logit_c)
    gW, gE, gW_c, gE_c = ref64.wnd_grad(rp, fid, fld, val, lab, W0, E0, Fc, d, pred, dz, l2, weights=weights,
                                        dz_cond=dz_c)
    _check_grad("W", W0, W1, gW, gW_c)
    _check_grad("E", E0, E1, gE, gE_c)
    live = np.ones(len(lab), bool) if weights is None else np.asarray(weights) != 0
    ent = np.repeat(live, np.diff(rp))
    _check_moved(W0, W1, E0, E1, d, fid[ent], v_fid=first[live][first[live] >= 0])
    for l, (got_w, got_b) in enumerate(dense or []):
        dW, db, dW_c, db_c = grads[l]
        for what, got, want, cond in (("dW", got_w, dW, dW_c), ("db", got_b, db, db_c)):
            ex = np.abs(got.astype(np.float64).ravel() - want.ravel()) - (1e-5 * cond.ravel() + 1e-30)
            at = int(np.argmax(ex))
            assert ex[at] <= 0, (what, l, float(ex[at]), at, float(got.ravel()[at]), float(want.ravel()[at]))


def _context(monkeypatch, Fc, d, hidden, act, l2):
    from lightctr_b200 import capi
    monkeypatch.setenv("LCTR_MLP_SKIP_UPDATE", "1")  # read when the context allocates its dense layers
    return _unit_sgd_context(capi.MODEL_WND, F, d, Fc, l2=l2, hidden=hidden, activation=act)


def _probe(monkeypatch, Fc, d, hidden, act, l2, batch, seed, ranges, weights=None):
    """the whole slot first (it sizes the source map, so every later range indexes inside it), then each row range"""
    W0, E0 = make_params(seed, F, d)
    dims = [Fc * d] + list(hidden) + [1]
    layers = wnd_layers(seed, dims)
    ctx = _context(monkeypatch, Fc, d, hidden, act, l2)
    for l, (w, b) in enumerate(layers):
        ctx.mlp_upload(l, w, b)
    rp, fid, fld, val, lab = batch
    ctx.upload_batch(0, rp, fid, fld, val, lab)
    if weights is not None:
        ctx.set_row_weights(0, weights)
    for i, (rb, re) in enumerate([(0, len(lab))] + list(ranges)):
        W1, E1, pred = _step(ctx, W0, E0, 0, rb, re)
        dense = [ctx.mlp_download_grad(l, dims[l], dims[l + 1]) for l in range(len(dims) - 1)] if i == 0 else None
        check_wnd(_rows(batch, rb, re), W0, E0, W1, E1, pred, Fc, d, layers, act, l2,
                  None if weights is None else weights[rb:re], dense)
    ctx.close()


def _apply_id(d):
    vec = 4 if d % 4 == 0 else 1
    lpr = 1
    while lpr < d // vec and lpr < 32:
        lpr <<= 1
    return f"apply_kernel-LPR{lpr}-VEC{vec}"


def _case_id(Fc, d):
    return f"wnd_forward_kernel-Fc{Fc}-seen{(Fc + 31) // 32}w-d{d}+wnd_backward_kernel+{_apply_id(d)}"


# (Fc, d, hidden, with_val): 1 to 64 bitmap words; d = 1, 3, 5 take the sparse apply's VEC 1 rows
SHAPES = [(1, 4, (16,), True), (13, 3, (16,), False), (32, 4, (16,), True), (33, 1, (16,), True),
          (39, 8, (12, 8), False), (64, 5, (16,), True), (2048, 1, (16,), False)]
ACTS = [pytest.param(0, id="sigmoid"), pytest.param(1, id="tanh")]
RANGES = [(5, 206), (1, 2), (150, 333)]  # sub-ranges: source map and dz rows indexed by r - rb


@pytest.mark.parametrize("act", ACTS)
@pytest.mark.parametrize("Fc,d,hidden,with_val", [pytest.param(*s, id=_case_id(s[0], s[1])) for s in SHAPES])
def test_wnd_gradient_vs_ref64(monkeypatch, Fc, d, hidden, with_val, act):
    """333 rows (not a multiple of the forward's 8 rows per CTA), then three sub-ranges starting at rb > 0; l2 = 1e-3"""
    seed = 7000 + Fc * 10 + d
    _probe(monkeypatch, Fc, d, hidden, act, 1e-3, wnd_batch(seed, Fc, 333, with_val), seed, RANGES)


@pytest.mark.parametrize("l2", [pytest.param(0.0, id="l2-0"), pytest.param(5e-2, id="l2-0.05")])
@pytest.mark.parametrize("Fc,d", [pytest.param(13, 3, id=_case_id(13, 3)), pytest.param(2048, 1, id=_case_id(2048, 1))])
def test_wnd_l2_on_wide_weights_only_vs_ref64(monkeypatch, Fc, d, l2):
    """L2 applies to the wide weights of every entry and never to the tensors: at 5e-2 an l2 E term is far outside the
    bound"""
    seed = 7500 + Fc + d
    _probe(monkeypatch, Fc, d, (16,), 0, l2, wnd_batch(seed, Fc, 333, True), seed, RANGES[:1])


@pytest.mark.parametrize("Fc,d", [pytest.param(Fc, d, id=_case_id(Fc, d).replace("backward_kernel", "backward_kernel-RW"))
                                  for Fc, d in ((13, 3), (39, 8))])
def test_wnd_weighted_rows_vs_ref64(monkeypatch, Fc, d):
    """row weights 0, fractional, integer, and one row whose weighted head w (p - y) passes the dense layers' +-15 clip
    (the wide gradient takes it unclipped); l2 = 5e-2, so the L2 term's weight w l2 shows"""
    seed = 7700 + Fc + d
    batch = wnd_batch(seed, Fc, 333, True)
    rng = np.random.default_rng(seed)
    weights = np.choose(rng.integers(0, 3, 333), [np.zeros(333), 0.25 + 0.5 * rng.random(333),
                                                  rng.integers(1, 4, 333).astype(np.float64)]).astype(np.float32)
    big = int(np.flatnonzero(np.diff(batch[0]) > 20)[0])
    weights[big] = 200.0
    weights[:4] = (0.0, 0.5, 3.0, 1.0)
    W0, E0 = make_params(seed, F, d)
    rp, fid, fld, val, lab = batch
    z, _f, wide, _zc, _wc = ref64.wnd_forward(rp, fid, fld, val, W0, E0, Fc, d)
    p64 = ref64.nfm_head(z, wide, wnd_layers(seed, [Fc * d, 16, 1]), 0, None, lab)[0]
    assert abs(weights[big] * (p64[big] - lab[big])) > 15
    _probe(monkeypatch, Fc, d, (16,), 0, 5e-2, batch, seed, RANGES[:1], weights)


def test_wnd_predict_and_score_vs_ref64():
    """wnd_forward_kernel + the fp32 forward-only chain on a slot of 2 * 65 536 + 123 rows: lctr_predict and lctr_score
    run it in score blocks of 65 536 rows, so every block after the first is a forward at rb > 0"""
    from lightctr_b200 import capi
    Fc, d, hidden, rows = 13, 4, (16,), 2 * 65536 + 123
    rng = np.random.default_rng(7900)
    lens = rng.integers(0, 20, rows)
    lens[rng.choice(rows, 200, replace=False)] = rng.choice([33, 65], 200)
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fid = rng.integers(0, F, rp[-1]).astype(np.uint32)
    fld = rng.integers(0, Fc, rp[-1]).astype(np.uint16)
    lab = (rng.random(rows) < 0.4).astype(np.int32)
    W0, E0 = make_params(7900, F, d)
    layers = wnd_layers(7900, [Fc * d] + list(hidden) + [1])
    ctx = capi.Context(capi.MODEL_WND, F, d, Fc, hidden=hidden)
    ctx.upload_params(W0, E0)
    for l, (w, b) in enumerate(layers):
        ctx.mlp_upload(l, w, b)
    ctx.upload_batch(0, rp, fid, fld, None, lab)
    z, _first, wide, z_c, w_c = ref64.wnd_forward(rp, fid, fld, None, W0, E0, Fc, d)
    p64, _dz, _dzc, logit_c = ref64.nfm_head(z, wide, layers, 0, None, lab, z_c, w_c)
    _check_pctr(ctx.predict(0), p64, logit_c)
    _check_pctr(ctx.score(0), p64, logit_c)
    ctx.close()
