"""Every FM / NFM / FFM kernel instantiation the launchers reach, checked against tests/ref64.py (float64, from the
definitions) or, for training steps, against the CPU oracle.  Each test id names the kernel and its template shape.

Batches (kernel_shapes_worker.make_batch): F = 4000, 300 rows of 0, 1, 63, 64, 65, 129, 300 and 2..40 entries, ids shared by
most rows, values != 1 or absent.

Forward bounds are condition-scaled: for the logit |z - z64| <= 1e-5 * cond + 1e-6, cond = sum of |w x| + 0.5 sum |x v|^2
+ 0.5 |sum |x v||^2 (ref64's figure), carried to the pCTR through the sigmoid's slope plus 3e-7 for the fp32 sigmoid; for
sumVX |s - s64| <= 1e-5 * sum |x v| + 1e-7.  A dropped or double-counted factor moves the logit by O(|V|^2) per pair, orders
of magnitude past these bounds."""
import os
import subprocess
import sys

import numpy as np
import pytest

import ref64
from conftest import ROOT
from kernel_shapes_worker import make_batch, make_params, run

pytestmark = pytest.mark.gpu

WORKER = os.path.join(ROOT, "tests", "kernel_shapes_worker.py")
F = 4000


def _rel(a, b):
    return abs(a - b) / max(abs(b), 1e-30)


def _within(got, want, cond, rtol=1e-5, atol=1e-7):
    err = np.abs(np.asarray(got, np.float64) - want)
    excess = err - (rtol * cond + atol)
    return float(excess.max()) <= 0, float(excess.max()), int(np.argmax(excess))


def _check_pctr(pctr, p64, z_cond):
    ok, ex, at = _within(pctr, p64, p64 * (1 - p64) * (1e-5 * z_cond + 1e-6), rtol=1.0, atol=3e-7)
    assert ok, ("pctr", ex, at, float(pctr[at]), float(p64[at]))


def _check_sumvx(sumvx, s64, s_cond):
    ok, ex, at = _within(sumvx.reshape(s64.shape), s64, s_cond)
    assert ok, ("sumvx", ex, divmod(at, s64.shape[1]))


def _inputs(model, k, Fc, det, batch, states, train, lr=0.05):
    rp, fid, fld, val, lab = batch
    d = dict(model=model, k=k, Fc=Fc, det=det, lr=lr, train=int(train), rp=rp, fid=fid, fld=fld, lab=lab,
             val=np.zeros(0, np.float32) if val is None else val)
    for i, st in enumerate(states):
        d[f"W{i}"], d[f"V{i}"] = st[0], st[1]
        if len(st) > 2:
            d[f"S{i}"] = st[2]
    return d


def _run_with_env(tmp_path, inp, env):
    src, dst = str(tmp_path / "in.npz"), str(tmp_path / "out.npz")
    np.savez(src, **inp)
    p = subprocess.run([sys.executable, WORKER, src, dst], env=dict(os.environ, **env), stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, timeout=600)
    assert p.returncode == 0, p.stdout
    with np.load(dst) as z:
        return {n: z[n] for n in z.files}


def _fwd_kind(k):
    return "coalesced" if k % 8 == 0 else "plain"


# ------------------------------------------------------------------------------------------------------------------------
# in-order FM forward (fm.cu fwd_go<K>): every instantiated K, through a parity-mode (deterministic = 1) predictor
# ------------------------------------------------------------------------------------------------------------------------
FWD_KS = [1, 2, 3, 4, 5, 6, 7, 8, 10, 12, 16, 20, 24, 32]


@pytest.mark.parametrize("with_val", [False, True], ids=["noval", "val"])
@pytest.mark.parametrize("k", [pytest.param(k, id=f"fwd_go-K{k}-{_fwd_kind(k)}") for k in FWD_KS])
def test_inorder_forward_vs_ref64(k, with_val):
    from lightctr_b200 import capi
    seed = 10 + k
    rp, fid, fld, val, lab = make_batch(seed, F, with_val=with_val)
    W, V = make_params(seed, F, k)
    out = run(_inputs(capi.MODEL_FM, k, 0, 1, (rp, fid, fld, val, lab), [(W, V)], train=False))
    s64, _z64, p64, s_c, z_c = ref64.fm_forward(rp, fid, val, W, V, k)
    _check_sumvx(out["sumvx0"], s64, s_c)
    _check_pctr(out["pctr0"], p64, z_c)


@pytest.mark.parametrize("with_val", [False, True], ids=["noval", "val"])
@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_forward_coalesced_kernel-K{k}") for k in (8, 16, 24, 32)])
def test_coalesced_forward_equals_plain_forward(tmp_path, k, with_val):
    """fm_forward_coalesced_kernel and fm_forward_kernel claim one expression sequence: pCTR and sumVX bit for bit."""
    from lightctr_b200 import capi
    seed = 50 + k
    batch = make_batch(seed, F, with_val=with_val)
    inp = _inputs(capi.MODEL_FM, k, 0, 1, batch, [make_params(seed, F, k)], train=False)
    co = run(inp)
    plain = _run_with_env(tmp_path, inp, {"LCTR_FWD_COALESCED": "0"})
    assert np.array_equal(co["sumvx0"].view(np.uint32), plain["sumvx0"].view(np.uint32))
    assert np.array_equal(co["pctr0"].view(np.uint32), plain["pctr0"].view(np.uint32))


# ------------------------------------------------------------------------------------------------------------------------
# dense gradient path (deterministic = 0, k not in {4, 8, 16, 32}): fm_backward_kernel<LPR, 1> + the sparse apply
# ------------------------------------------------------------------------------------------------------------------------
DENSE_FM = [(1, 1), (2, 2), (3, 4), (6, 8), (12, 16), (24, 32)]  # (k, LPR)


def _params_close(got, want, tol, threshold_updater):
    """max |got - want| < tol; FTRL's hard threshold (|z| <= lambda1 -> w = 0) may put a coordinate whose z is within
    rounding of lambda1 on the other side: at most 1e-5 of them, each by at most one such jump (1e-2)."""
    d = np.abs(got - want)
    if not threshold_updater:
        return float(d.max()) < tol
    return float(np.mean(d > tol)) <= 1e-5 and float(d.max()) < 1e-2


@pytest.mark.parametrize("opt", ["adagrad", "ftrl"])
@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_kernel-LPR{l}-K{k}") for k, l in DENSE_FM])
def test_dense_path_fm_step_vs_oracle(oracle_api, k, opt):
    """Two steps, each from the oracle's exact state (parameters + updater state): the loss within 1e-6 and the
    parameters within 2e-5, the tolerances of the order-free step's test."""
    from lightctr_b200 import capi
    seed = 100 + k
    rp, fid, fld, val, lab = make_batch(seed, F, with_val=k % 2 == 0)
    W0, V0 = make_params(seed, F, k)
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32) if val is None else val, lab, F, 0)
    o = oracle_api.FMOracle(ds, k, W0, V0)
    o.opt = opt
    ctx = capi.Context(capi.MODEL_FM, F, k, optimizer={"adagrad": capi.OPT_ADAGRAD, "ftrl": capi.OPT_FTRL}[opt],
                       deterministic=0)
    ctx.upload_params(W0, V0)
    ctx.upload_batch(0, rp, fid, None, val, lab)
    F1 = F * (k + 1)
    for step in range(2):
        if step > 0:
            ctx.upload_params(o.W, o.V)
            ctx.upload_opt_state(o.accum, getattr(o, "s2", np.zeros(F1, np.float32)))
        lg, cg = ctx.train_step(0)
        lo, ao = o.epoch()
        assert _rel(lg, lo) < 1e-6, (step, lg, lo)
        assert abs(cg - round(ao * len(lab))) <= 1
        Wg, Vg = ctx.download_params()
        thr = opt == "ftrl"
        assert _params_close(Wg, o.W, 2e-5, thr) and _params_close(Vg, o.V, 2e-5, thr), step
    ctx.close()


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_kernel-NFM-LPR{l}-K{k}") for k, l in DENSE_FM if k in (6, 12, 24)])
def test_dense_path_nfm_step_vs_oracle(oracle_api, k):
    _nfm_step_vs_oracle(oracle_api, k, det=0, seed=300 + k)


def _nfm_step_vs_oracle(oracle_api, k, det, seed):
    """One minibatch from identical state (dropout masks 1, Adagrad state 1 so that the first step is linear in g rather
    than sign-like): loss within 1e-5 (fp32 dense layers), W and V within 2e-5."""
    from lightctr_b200 import capi
    rp, fid, fld, val, lab = make_batch(seed, F, with_val=True)
    W0, V0 = make_params(seed, F, k)
    rows, H = len(lab), 16
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), val, lab, F, 0)
    o = oracle_api.NFMOracle(ds, k, [H], W=W0, V=V0, batch_size=rows, minibatch=rows)
    o.accum[:] = 1.0
    layers = []
    for l in range(2):
        o.mlp.arrays("mask", l)[:] = 1.0
        layers.append((o.mlp.arrays("weight", l).copy(), o.mlp.arrays("bias", l).copy()))
    ctx = capi.Context(capi.MODEL_NFM, F, k, hidden=(H,), minibatch_size=rows, deterministic=det,
                       csc_row_block=rows if det else 0)
    ctx.upload_params(W0, V0)
    ctx.upload_opt_state(np.ones(F * (k + 1), np.float32))
    for l, (w, b) in enumerate(layers):
        ctx.mlp_upload(l, w, b)
    ctx.upload_batch(0, rp, fid, None, val, lab)
    lg, _ = ctx.train_step(0)
    lo, _ = o.epoch()
    assert _rel(lg, lo) < 1e-5, (lg, lo)
    Wg, Vg = ctx.download_params()
    assert np.max(np.abs(Wg - o.W)) < 2e-5 and np.max(np.abs(Vg - o.V)) < 2e-5
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------
# feature-major backward (deterministic = 1): fm_backward_csc_kernel<LR>, LR = 4 (k <= 4), 8, 16, 32 (k = 17..32)
# ------------------------------------------------------------------------------------------------------------------------
CSC = [(3, 4), (4, 4), (20, 32), (24, 32), (32, 32)]  # (k, LR)


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_csc_kernel-LR{l}-K{k}") for k, l in CSC])
def test_feature_major_fm_steps_vs_oracle(oracle_api, k):
    """Three steps in a row (no re-sync): the loss within the 1e-5 bar, parameters within 1e-5."""
    from lightctr_b200 import capi
    seed = 400 + k
    rp, fid, fld, val, lab = make_batch(seed, F, with_val=k % 2 == 1)
    W0, V0 = make_params(seed, F, k)
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32) if val is None else val, lab, F, 0)
    o = oracle_api.FMOracle(ds, k, W0, V0)
    ctx = capi.Context(capi.MODEL_FM, F, k, deterministic=1)
    ctx.upload_params(W0, V0)
    ctx.upload_batch(0, rp, fid, None, val, lab)
    for step in range(3):
        lg, _ = ctx.train_step(0)
        lo, _ = o.epoch()
        assert _rel(lg, lo) < 1e-5, (step, lg, lo)
    W, V = ctx.download_params()
    assert np.max(np.abs(W - o.W)) < 1e-5 and np.max(np.abs(V - o.V)) < 1e-5
    ctx.close()


@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_backward_csc_kernel-NFM-LR{l}-K{k}") for k, l in CSC])
def test_feature_major_nfm_step_vs_oracle(oracle_api, k):
    _nfm_step_vs_oracle(oracle_api, k, det=1, seed=500 + k)


# ------------------------------------------------------------------------------------------------------------------------
# CTA-per-sample FFM kernel (ffm.cu ffm_fused_kernel<VEC>): k % 4 != 0 always, k % 4 == 0 with LCTR_FFM_WARP=0
# ------------------------------------------------------------------------------------------------------------------------
def _vec(k):
    return 4 if k % 4 == 0 else (2 if k % 2 == 0 else 1)


FFM_CTA = [(5, 2, True), (13, 6, False), (7, 3, True), (39, 1, False)]


@pytest.mark.parametrize("Fc,k,with_val", [pytest.param(Fc, k, v, id=f"ffm_fused_kernel-VEC{_vec(k)}-Fc{Fc}-K{k}")
                                           for Fc, k, v in FFM_CTA])
def test_ffm_cta_kernel_vs_oracle_and_ref64(oracle_api, Fc, k, with_val):
    _ffm_cta_check(oracle_api, Fc, k, with_val, seed=600 + Fc * 10 + k, runner=run)


@pytest.mark.parametrize("Fc,k", [pytest.param(39, 4, id="ffm_fused_kernel-VEC4-Fc39-K4-LCTR_FFM_WARP0")])
def test_ffm_cta_kernel_vec4_without_the_warp_kernel(oracle_api, tmp_path, Fc, k):
    """Training at Fc <= 64 with k % 4 == 0 goes to the warp kernel unless LCTR_FFM_WARP=0: the CTA kernel's VEC = 4
    instantiation at such a field count runs in a process of its own."""
    _ffm_cta_check(oracle_api, Fc, k, True, seed=700,
                   runner=lambda inp: _run_with_env(tmp_path, inp, {"LCTR_FFM_WARP": "0"}))


def _ffm_cta_check(oracle_api, Fc, k, with_val, seed, runner):
    """Two training steps, each from the oracle's exact state (loss within the 1e-5 bar, parameters within 2e-5, correct
    count within 1), then the order-free predictor against ref64's pair loop."""
    from lightctr_b200 import capi
    rp, fid, fld, val, lab = make_batch(seed, F, Fc=Fc, with_val=with_val)
    W0, V0 = make_params(seed, F, k, Fc)
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32) if val is None else val, lab, F, Fc)
    o = oracle_api.FFMOracle(ds, k, W0, V0)
    states, want = [], []
    for _ in range(2):
        states.append((o.W.copy(), o.V.copy(), o.s1.copy()))
        want.append(o.epoch() + (o.W.copy(), o.V.copy()))
    batch = (rp, fid, fld, val, lab)
    got = runner(_inputs(capi.MODEL_FFM, k, Fc, 0, batch, states, train=True))
    for i, (lo, ao, Wo, Vo) in enumerate(want):
        assert _rel(float(got[f"loss{i}"]), lo) < 1e-5, (i, float(got[f"loss{i}"]), lo)
        assert abs(float(got[f"cnt{i}"]) - round(ao * len(lab))) <= 1
        assert np.max(np.abs(got[f"Wout{i}"] - Wo)) < 2e-5 and np.max(np.abs(got[f"Vout{i}"] - Vo)) < 2e-5, i
    pr = runner(_inputs(capi.MODEL_FFM, k, Fc, 0, batch, [(W0, V0)], train=False))
    _z, p64, z_c = ref64.ffm_forward(rp, fid, fld, val, W0, V0, Fc, k)
    _check_pctr(pr["pctr0"], p64, z_c)


# ------------------------------------------------------------------------------------------------------------------------
# order-free FM predictor (fm_fused.cuh fm_fused_kernel MODE 0): deterministic = 0 at k in {4, 8, 16, 32}
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("with_val", [False, True], ids=["noval", "val"])
@pytest.mark.parametrize("k", [pytest.param(k, id=f"fm_fused_kernel-MODE0-K{k}") for k in (4, 8, 16, 32)])
def test_order_free_predictor_vs_ref64(k, with_val):
    from lightctr_b200 import capi
    seed = 800 + k
    rp, fid, fld, val, lab = make_batch(seed, F, with_val=with_val)
    W, V = make_params(seed, F, k)
    out = run(_inputs(capi.MODEL_FM, k, 0, 0, (rp, fid, fld, val, lab), [(W, V)], train=False))
    s64, _z, p64, s_c, z_c = ref64.fm_forward(rp, fid, val, W, V, k)
    _check_sumvx(out["sumvx0"], s64, s_c)
    _check_pctr(out["pctr0"], p64, z_c)


# ------------------------------------------------------------------------------------------------------------------------
# refusals: an error with the launcher's message, and the device still trains a second context afterwards
# ------------------------------------------------------------------------------------------------------------------------
def _still_trains(oracle_api):
    from lightctr_b200 import capi
    rp, fid, fld, val, lab = make_batch(900, F, with_val=False)
    W0, V0 = make_params(900, F, 8)
    ctx = capi.Context(capi.MODEL_FM, F, 8, deterministic=1)
    ctx.upload_params(W0, V0)
    ctx.upload_batch(0, rp, fid, None, None, lab)
    lg, _ = ctx.train_step(0)
    ctx.close()
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), np.ones(len(fid), np.float32), lab, F, 0)
    lo, _ = oracle_api.FMOracle(ds, 8, W0, V0).epoch()
    assert _rel(lg, lo) < 1e-5, (lg, lo)


def _tiny(Fc):
    rp = np.array([0, 3, 5], np.int64)
    return rp, np.array([1, 2, 3, 4, 5], np.uint32), (np.arange(5) % max(Fc, 1)).astype(np.uint16), np.array([1, 0], np.int32)


@pytest.mark.parametrize("Fc,k,msg", [pytest.param(1100, 1, "exceeds one CTA", id="ffm-A1100-past-1024-slots"),
                                      pytest.param(100, 8, "needs .* shared memory", id="ffm-Fc100-K8-past-227KB")])
def test_ffm_shape_past_the_kernel_is_refused(oracle_api, Fc, k, msg):
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_FFM, 10, k, Fc)
    rp, fid, fld, lab = _tiny(Fc)
    ctx.upload_batch(0, rp, fid, fld, None, lab)
    with pytest.raises(capi.LctrError, match=msg):
        ctx.train_step(0)
    with pytest.raises(capi.LctrError, match=msg):
        ctx.predict(0)
    ctx.close()
    _still_trains(oracle_api)


@pytest.mark.parametrize("det", [0, 1])
def test_fm_k_not_instantiated_is_refused(oracle_api, det):
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_FM, 10, 9, deterministic=det)
    rp, fid, _fld, lab = _tiny(0)
    ctx.upload_batch(0, rp, fid, None, None, lab)
    with pytest.raises(capi.LctrError, match="factor_cnt=9 is not instantiated"):
        ctx.train_step(0)
    with pytest.raises(capi.LctrError, match="factor_cnt=9 is not instantiated"):
        ctx.predict(0)
    ctx.close()
    _still_trains(oracle_api)


def test_nfm_device_grouped_upload_is_refused(oracle_api):
    from lightctr_b200 import capi
    ctx = capi.Context(capi.MODEL_NFM, 10, 8, hidden=(4,), deterministic=2)
    rp, fid, _fld, lab = _tiny(0)
    with pytest.raises(capi.LctrError, match="deterministic=2 .* needs FM with k in"):
        ctx.upload_batch(0, rp, fid, None, None, lab)
    ctx.close()
    _still_trains(oracle_api)
