"""The per-feature gradient of every FM / NFM / FFM training path, recovered from one unit SGD step and held against
tests/ref64.py.  Each test id names the kernel and its template shape.

The probe: a context with the parameter-server SGD rule (OPT_PS_SGD), which steps w -= g / (mb / lr), and lr = mb
(minibatch_size, or the rows of the step when it is 0), so the divisor is exactly 1 and g = w0 - w1 up to the rounding of
w1.  Unlike an Adagrad step from a zero state (which moves every coordinate with |g / B| >~ 3e-3 by +-lr), this shows the
size of every coordinate's gradient, the heavy ones included.  Checks, per step:
- |g - g64| <= 1e-5 * cond + spacing(w1) (ref64.probe_excess), with ref64's gradient and condition figure evaluated at the
  kernel's own pCTR, which is itself held to ref64's forward;
- exactly the ids of the rows stepped moved (W), and no V row outside them.
NFM: ref64.nfm_head restates the dense layers; the error of the fp32 dz is folded into gV's condition.  Wide&Deep has
tests/test_wnd_gpu.py, which shares these checks.
Two ranks on one device: the merged shards against ref64 on the concatenated batch and the concatenated per-rank pCTR."""
import os
import subprocess
import sys

import numpy as np
import pytest

import multirank as mr
import ref64
from conftest import ROOT
from kernel_shapes_worker import make_batch, make_params, run

pytestmark = pytest.mark.gpu

WORKER = os.path.join(ROOT, "tests", "kernel_shapes_worker.py")
L2 = 0.001


# ------------------------------------------------------------------------------------------------------------------------
# checks
# ------------------------------------------------------------------------------------------------------------------------
def _check_pctr(pctr, p64, z_cond):
    err = np.abs(pctr.astype(np.float64) - p64)
    ex = err - (p64 * (1 - p64) * (1e-5 * z_cond + 1e-6) + 3e-7)
    at = int(np.argmax(ex)) if len(ex) else 0
    assert not len(ex) or ex[at] <= 0, ("pctr", float(ex[at]), at, float(pctr[at]), float(p64[at]))


def _check_grad(what, w0, w1, g64, cond):
    got = w0.astype(np.float64) - w1.astype(np.float64)
    ex = ref64.probe_excess(got, g64.ravel(), cond.ravel(), w1)
    at = int(np.argmax(ex))
    assert ex[at] <= 0, (what, float(ex[at]), at, float(got[at]), float(g64.ravel()[at]), float(cond.ravel()[at]))


def _check_moved(W0, W1, V0, V1, rowlen, fid, exact_v=True, v_fid=None):
    """W moved on exactly the ids of fid; V on exactly those of v_fid (default fid), or only inside them (exact_v False)"""
    ids = np.unique(fid)
    v_ids = ids if v_fid is None else np.unique(v_fid)
    moved_w = np.flatnonzero(W1 != W0)
    moved_v = np.flatnonzero(np.any((V1 != V0).reshape(-1, rowlen), 1))
    assert np.array_equal(moved_w, ids), ("W moved", len(moved_w), len(ids), np.setxor1d(moved_w, ids)[:8])
    assert np.all(np.isin(moved_v, v_ids)), ("V moved outside the batch", np.setdiff1d(moved_v, v_ids)[:8])
    if exact_v:
        assert np.array_equal(moved_v, v_ids), ("V rows that did not move", np.setdiff1d(v_ids, moved_v)[:8])


def _rows(batch, rb, re):
    rp, fid, fld, val, lab = batch
    b, e = rp[rb], rp[re]
    return (rp[rb:re + 1] - b, fid[b:e], fld[b:e], None if val is None else val[b:e], lab[rb:re])


def _check_fm(sub, W0, V0, W1, V1, pred, k, l2=L2):
    rp, fid, _fld, val, lab = sub
    s64, _z, p64, _sc, z_c = ref64.fm_forward(rp, fid, val, W0, V0, k)
    _check_pctr(pred, p64, z_c)
    gW, gV, gW_c, gV_c = ref64.fm_grad(rp, fid, val, lab, W0, V0, k, pred, s64, l2)
    _check_grad("W", W0, W1, gW, gW_c)
    _check_grad("V", V0, V1, gV, gV_c)
    _check_moved(W0, W1, V0, V1, k, fid)


def _check_nfm(sub, W0, V0, W1, V1, pred, k, layers, l2=L2):
    rp, fid, _fld, val, lab = sub
    z, wide, s64, z_c, w_c = ref64.nfm_forward(rp, fid, val, W0, V0, k)
    p64, dz, dz_c, logit_c = ref64.nfm_head(z, wide, layers, 0, None, lab, z_c, w_c)
    _check_pctr(pred, p64, logit_c)
    gW, gV, gW_c, gV_c = ref64.nfm_grad(rp, fid, val, lab, W0, V0, k, pred, s64, dz, l2, dz_cond=dz_c)
    _check_grad("W", W0, W1, gW, gW_c)
    _check_grad("V", V0, V1, gV, gV_c)
    _check_moved(W0, W1, V0, V1, k, fid)


def _check_ffm(batch, W0, V0, W1, V1, pred, Fc, k, l2):
    rp, fid, fld, val, lab = batch
    _z, p64, z_c = ref64.ffm_forward(rp, fid, fld, val, W0, V0, Fc, k)
    _check_pctr(pred, p64, z_c)
    gW, gV, gW_c, gV_c = ref64.ffm_grad(rp, fid, fld, val, lab, W0, V0, Fc, k, pred, l2)
    _check_grad("W", W0, W1, gW, gW_c)
    _check_grad("V", V0, V1, gV, gV_c)
    # a slot V[f, b] moves only when some pair of f's rows reaches field b
    _check_moved(W0, W1, V0, V1, Fc * k, fid, exact_v=False)


# ------------------------------------------------------------------------------------------------------------------------
# probes
# ------------------------------------------------------------------------------------------------------------------------
def _unit_sgd_context(model, F, k, Fc=0, l2=L2, **kw):
    """a context whose step is w -= g: OPT_PS_SGD with minibatch_size = lr = 1"""
    from lightctr_b200 import capi
    return capi.Context(model, F, k, Fc, optimizer=capi.OPT_PS_SGD, lr=1.0, minibatch_size=1, l2=l2, **kw)


def _step(ctx, W0, V0, slot, rb, re):
    ctx.upload_params(W0, V0)
    ctx.train_step(slot, rb, re)
    W1, V1 = ctx.download_params()
    return W1, V1, ctx.download_pred(slot)[rb:re]


def _run_with_env(tmp_path, inp, env):
    src, dst = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    np.savez(src, **inp)
    p = subprocess.run([sys.executable, WORKER, src, dst], env=dict(os.environ, **env), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout
    with np.load(dst) as z:
        return {n: z[n] for n in z.files}


def _worker_probe(model, k, Fc, det, batch, W0, V0, l2, env=None, tmp_path=None):
    """one unit SGD step through kernel_shapes_worker.run (in a process of its own when env is given):
    returns W1, V1 and the step's pCTR"""
    from lightctr_b200 import capi
    rp, fid, fld, val, lab = batch
    inp = dict(model=model, k=k, Fc=Fc, det=det, lr=1.0, train=1, rp=rp, fid=fid, fld=fld, lab=lab,
               val=np.zeros(0, np.float32) if val is None else val, opt=capi.OPT_PS_SGD, l2=l2, mb=1, W0=W0, V0=V0)
    out = run(inp) if env is None else _run_with_env(tmp_path, inp, env)
    return out["Wout0"], out["Vout0"], out["pred0"]


# ------------------------------------------------------------------------------------------------------------------------
# batches of the order-free step
# ------------------------------------------------------------------------------------------------------------------------
def _npass(k):
    return 8 if k <= 8 else (4 if k == 16 else 2)  # fm_fused_kernel's 32-entry register passes


def compact_batch(seed, F, k, rows, n_cand, with_val):
    """Rows for fm_fused_kernel's hot-slot map (an id is hot with max(3, ceil(128 * 512 / rows)) hits in the first 512
    rows: 4 at 16 384 rows; at most kHotMax = 2048 ids are):
    - id 0 in every non-empty row;
    - ids 1..n_cand four times each in the first 512 rows, and two of them in every later row;
    - id n_cand + 1 in every row of the first 512 with more than one entry, and in no later row;
    - id n_cand + 2 in none of the first 512 rows and in every later row with more than one entry;
    - rows of NPASS*32 - 1, NPASS*32, NPASS*32 + 1, 0 and 1 entries, inside and after the first 512 rows;
    - the rest 2..12 entries from the ids above n_cand + 2, in random order."""
    rng = np.random.default_rng(seed)
    sampled = min(rows, 512)
    cand, early, late = np.arange(1, n_cand + 1), n_cand + 1, n_cand + 2
    np_ = _npass(k)
    special = {}
    for base in (7, sampled + 7):
        if base + 5 <= rows:
            for j, n in enumerate((np_ * 32 - 1, np_ * 32, np_ * 32 + 1, 0, 1)):
                special[base + j] = n
    ids = [[] for _ in range(rows)]
    free = np.array([r for r in range(sampled) if r not in special])
    for h in cand:
        for r in rng.choice(free, 4, replace=False):
            ids[r].append(h)
    out = []
    for r in range(rows):
        n = special.get(r)
        if n == 0:
            out.append(np.zeros(0, np.int64))
            continue
        row = [0] if n == 1 else [0, early if r < sampled else late] + ids[r]
        if r >= sampled and n is None:
            row += list(rng.choice(cand, 2, replace=False))
        if n is None:
            extra = np.unique(rng.integers(n_cand + 3, F, int(rng.integers(2, 13))))
        else:
            extra = rng.choice(np.arange(n_cand + 3, F), n - len(row), replace=False)
        out.append(rng.permutation(np.concatenate([np.asarray(row, np.int64), extra.astype(np.int64)])))
    lens = np.array([len(o) for o in out])
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fid = np.concatenate(out).astype(np.uint32)
    fld = np.zeros(len(fid), np.uint16)
    val = (0.25 + 1.5 * rng.random(len(fid))).astype(np.float32) if with_val else None
    lab = (rng.random(rows) < 0.4).astype(np.int32)
    return rp, fid, fld, val, lab


def _upload(ctx, slot, batch):
    rp, fid, _fld, val, lab = batch
    ctx.upload_batch(slot, rp, fid, None, val, lab)


# ------------------------------------------------------------------------------------------------------------------------
# FM, dense path: fm_backward_kernel<LPR, 1> + the sparse apply (k not in {4, 8, 16, 32})
# ------------------------------------------------------------------------------------------------------------------------
DENSE_FM = [(1, 1), (2, 2), (3, 4), (6, 8), (12, 16), (24, 32)]  # (k, LPR)


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_kernel-LPR{l}-K{k}") for k, l in DENSE_FM])
def test_dense_path_fm_gradient_vs_ref64(k):
    """lr = B with minibatch_size 0: the divisor B / lr is exactly 1."""
    from lightctr_b200 import capi
    seed = 200 + k
    F = 4000
    batch = make_batch(seed, F, with_val=True)
    rp, fid, fld, val, lab = batch
    W0, V0 = make_params(seed, F, k)
    ctx = capi.Context(capi.MODEL_FM, F, k, optimizer=capi.OPT_PS_SGD, deterministic=0, lr=float(len(lab)))
    ctx.upload_params(W0, V0)
    ctx.upload_batch(0, rp, fid, None, val, lab)
    ctx.train_step(0)
    W1, V1 = ctx.download_params()
    pred = ctx.download_pred(0)
    ctx.close()
    _check_fm(batch, W0, V0, W1, V1, pred, k)


# ------------------------------------------------------------------------------------------------------------------------
# FM, order-free step: fm_fused_kernel MODE 1 + apply_compact_kernel (deterministic = 0, k in {4, 8, 16, 32})
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_val", [False, True], ids=["noval", "val"])
@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_fused_kernel-MODE1-NPASS{_npass(k)}-K{k}+apply_compact_kernel")
                               for k in (4, 8, 16, 32)])
def test_compact_fm_gradient_vs_ref64(k, with_val):
    """16 384 rows with more than kHotMax = 2048 hot candidates (so the hot map is full and the rest stay ordinary slots):
    the whole slot; a second slot whose ids overlap the first in part and whose hot set differs (a G / Ghot row the first
    step left non-zero shows up here); then row ranges of the first slot, across the sampled rows' end."""
    from lightctr_b200 import capi
    F = 60000
    big = compact_batch(1000 + k, F, k, 16384, 2200, with_val)
    small = compact_batch(2000 + k, F, k, 600, 100, with_val)
    W0, V0 = make_params(3000 + k, F, k)
    ctx = _unit_sgd_context(capi.MODEL_FM, F, k, deterministic=0)
    _upload(ctx, 0, big)
    _upload(ctx, 1, small)
    for slot, batch, rb, re in ((0, big, 0, 16384), (1, small, 0, 600), (0, big, 0, 1), (0, big, 300, 700),
                                (0, big, 15000, 16384)):
        W1, V1, pred = _step(ctx, W0, V0, slot, rb, re)
        _check_fm(_rows(batch, rb, re), W0, V0, W1, V1, pred, k)
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------
# NFM embedding backward: fm_fused_kernel MODE 3 + apply_compact_kernel; fm_backward_csc_kernel NFM (deterministic = 1)
# ------------------------------------------------------------------------------------------------------------------------
NFM_H = 16


def _nfm_layers(seed, k):
    rng = np.random.default_rng(seed)
    return [((rng.random((NFM_H, k)) - 0.5).astype(np.float32), (rng.standard_normal(NFM_H) * 0.1).astype(np.float32)),
            ((rng.random((1, NFM_H)) - 0.5).astype(np.float32), (rng.standard_normal(1) * 0.1).astype(np.float32))]


def _nfm_probe(k, det, batch, seed):
    from lightctr_b200 import capi
    F = 60000 if det == 0 else 4000
    W0, V0 = make_params(seed, F, k)
    layers = _nfm_layers(seed, k)
    rows = len(batch[4])
    ctx = _unit_sgd_context(capi.MODEL_NFM, F, k, hidden=(NFM_H,), deterministic=det, csc_row_block=rows if det else 0)
    for l, (w, b) in enumerate(layers):
        ctx.mlp_upload(l, w, b)
    _upload(ctx, 0, batch)
    W1, V1, pred = _step(ctx, W0, V0, 0, 0, rows)
    ctx.close()
    _check_nfm(batch, W0, V0, W1, V1, pred, k, layers)


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_fused_kernel-MODE3-NPASS{_npass(k)}-K{k}+apply_compact_kernel")
                               for k in (4, 8, 16, 32)])
def test_compact_nfm_gradient_vs_ref64(k):
    """2048 rows: ids 0 and 201 are hot (in every sampled row), the NPASS edges are there; fp32 dense layers, masks 1."""
    _nfm_probe(k, 0, compact_batch(4000 + k, 60000, k, 2048, 200, True), seed=4100 + k)


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_csc_kernel-NFM-LR{l}-K{k}") for k, l in ((3, 4), (12, 16), (24, 32))])
def test_feature_major_nfm_gradient_vs_ref64(k):
    _nfm_probe(k, 1, make_batch(4200 + k, 4000, with_val=True), seed=4300 + k)


# ------------------------------------------------------------------------------------------------------------------------
# FM feature-major: fm_backward_csc_kernel<LR> (deterministic = 1) and the device-grouped step (deterministic = 2)
# ------------------------------------------------------------------------------------------------------------------------
def _with_hot_id(batch, hot=0):
    """id `hot` in every non-empty row (it replaces the row's first entry where the row lacks it)"""
    rp, fid, fld, val, lab = batch
    fid = fid.copy()
    for r in range(len(lab)):
        b, e = rp[r], rp[r + 1]
        if e > b and not np.any(fid[b:e] == hot):
            fid[b] = hot
    return rp, fid, fld, val, lab


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_csc_kernel-LR{l}-K{k}") for k, l in ((3, 4), (6, 8), (12, 16), (24, 32))])
def test_feature_major_fm_gradient_vs_ref64(k):
    from lightctr_b200 import capi
    F = 4000
    batch = _with_hot_id(make_batch(5000 + k, F, with_val=k % 2 == 0))
    W0, V0 = make_params(5000 + k, F, k)
    W1, V1, pred = _worker_probe(capi.MODEL_FM, k, 0, 1, batch, W0, V0, L2)
    _check_fm(batch, W0, V0, W1, V1, pred, k)


@pytest.mark.parametrize("k", [pytest.param(8, id="fm_backward_devcsc-K8-feature-of-600-entries")])
def test_device_grouped_fm_gradient_vs_ref64(k):
    """deterministic = 2: the batch is grouped by feature on the device; id 0 has one entry per row (> 256)."""
    from lightctr_b200 import capi
    F = 4000
    batch = _with_hot_id(make_batch(5100, F, rows=600, with_val=True))
    W0, V0 = make_params(5100, F, k)
    W1, V1, pred = _worker_probe(capi.MODEL_FM, k, 0, 2, batch, W0, V0, L2)
    _check_fm(batch, W0, V0, W1, V1, pred, k)


# ------------------------------------------------------------------------------------------------------------------------
# FFM: ffm_warp_kernel<PASSES>, ffm_fused_kernel<VEC>, ffm_tma_kernel, the bulk-reduce variant and the grouped step
# ------------------------------------------------------------------------------------------------------------------------
FFM_L2 = [pytest.param(l2, id=f"l2-{l2:g}") for l2 in (0.0, 1e-3, 5e-2)]
FFM_WARP = [(6, 4), (39, 4), (39, 8), (33, 12), (64, 4)]  # (Fc, k): 1, 2, 3, 4, 2 passes of 32 slots


def _ffm_case(seed, Fc, k, with_val=True, rows=300, hot=False):
    F = 4000
    batch = make_batch(seed, F, rows=rows, Fc=Fc, with_val=with_val)
    if hot:
        batch = _with_hot_id(batch)
    return batch, make_params(seed, F, k, Fc)


@pytest.mark.parametrize("l2", FFM_L2)
@pytest.mark.parametrize("Fc,k", [pytest.param(Fc, k, id=f"ffm_warp_kernel-PASSES{(Fc * k // 4 + 31) // 32}-Fc{Fc}-K{k}")
                                  for Fc, k in FFM_WARP])
def test_ffm_warp_gradient_vs_ref64(Fc, k, l2):
    """rows with fields absent and entries of one field apart (make_batch's fields are random per entry); at l2 = 5e-2
    the l2 count c_ib of every slot is far above the bound"""
    from lightctr_b200 import capi
    batch, (W0, V0) = _ffm_case(6000 + Fc * 10 + k, Fc, k, with_val=Fc != 64)
    W1, V1, pred = _worker_probe(capi.MODEL_FFM, k, Fc, 0, batch, W0, V0, l2)
    _check_ffm(batch, W0, V0, W1, V1, pred, Fc, k, l2)


FFM_ENV = [
    pytest.param(7, 3, 0, {}, id="ffm_fused_kernel-VEC1-Fc7-K3"),
    pytest.param(13, 6, 0, {}, id="ffm_fused_kernel-VEC2-Fc13-K6"),
    pytest.param(39, 4, 0, {"LCTR_FFM_WARP": "0"}, id="ffm_fused_kernel-VEC4-Fc39-K4-LCTR_FFM_WARP0"),
    pytest.param(39, 4, 0, {"LCTR_FFM_TMA": "1", "LCTR_FFM_WARP": "0"}, id="ffm_tma_kernel-Fc39-K4"),
    pytest.param(39, 4, 0, {"LCTR_FFM_BULK": "1"}, id="ffm_fused_kernel-VEC4-bulk-Fc39-K4-LCTR_FFM_BULK1"),
    pytest.param(39, 4, 2, {}, id="ffm_grouped-Fc39-K4-feature-of-600-entries"),
]


@pytest.mark.parametrize("l2", [pytest.param(l2, id=f"l2-{l2:g}") for l2 in (1e-3, 5e-2)])
@pytest.mark.parametrize("Fc,k,det,env", FFM_ENV)
def test_ffm_other_kernels_gradient_vs_ref64(tmp_path, Fc, k, det, env, l2):
    """the CTA-per-sample kernel at VEC 1 / 2 / 4, the TMA-staged and bulk-reduce kernels (read from the environment once
    per process: a process of their own) and the grouped step (deterministic = 2, id 0 in each of 600 rows)"""
    from lightctr_b200 import capi
    batch, (W0, V0) = _ffm_case(6500 + Fc * 10 + k + det, Fc, k, with_val=k != 6, rows=600 if det == 2 else 300,
                                hot=det == 2)
    W1, V1, pred = _worker_probe(capi.MODEL_FFM, k, Fc, det, batch, W0, V0, l2, env=env or None, tmp_path=tmp_path)
    _check_ffm(batch, W0, V0, W1, V1, pred, Fc, k, l2)


# ------------------------------------------------------------------------------------------------------------------------
# two ranks on one device (CUDA IPC): push_rows_kernel's hot fold + merge_apply_kernel (FM / NFM), merge_kernel + the
# sparse apply (FFM)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("model,F,k,rows", [
    pytest.param("fm", 20000, 16, 2048, id="push_rows_kernel-hot+merge_apply_kernel-FM-K16"),
    pytest.param("nfm", 20000, 16, 1024, id="push_rows_kernel+merge_apply_kernel-NFM-K16"),
    pytest.param("ffm", 6000, 4, 256, id="merge_kernel+apply-FFM-Fc39-K4"),
    pytest.param("wnd", 20000, 4, 512, id="wnd_backward_kernel-ent_pslot+merge_kernel+apply-WND-Fc39-d4"),
])
def test_two_ranks_gradient_vs_ref64(tmp_path, model, F, k, rows):
    """lr = minibatch_size = the global batch; 2048 Criteo-shaped rows per rank put the frequent ids of the FM case over
    the hot threshold (32 hits in the first 512 rows)."""
    from lightctr_b200 import dist as ldist
    mr.launch("dist_worker.py", tmp_path, ["--mode", "gpu", "--same-device", "--probe", "--steps", "1", "--model", model,
                                           "--F", str(F), "--k", str(k), "--rows", str(rows)])
    parts = mr.load(tmp_path)
    W1 = ldist.merge_shards([p["W"] for p in parts], 2, F)
    V1 = ldist.merge_shards([p["V"] for p in parts], 2, F)
    pred = np.concatenate([p["pred"] for p in parts])
    W0, V0 = mr.make_params(F, k, model)
    rp, fid, fld, lab = mr.global_batch([mr.train_batches(F, rows, 1, r)[0] for r in range(2)])
    batch = (rp, fid, fld, None, lab)
    if model == "fm":
        _check_fm(batch, W0, V0, W1, V1, pred, k)
    elif model == "nfm":
        _check_nfm(batch, W0, V0, W1, V1, pred, k, mr.dense_layers(model, k))
    elif model == "wnd":  # every rank's own dense layers, equal at the first step
        from test_wnd_gpu import check_wnd
        check_wnd(batch, W0, V0, W1, V1, pred, 39, k, mr.dense_layers(model, k), 0, L2)
    else:
        _check_ffm(batch, W0, V0, W1, V1, pred, 39, k, L2)
