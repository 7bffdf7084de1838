"""lctr_score (include/lightctr_b200.h): the forward half of lctr_train_step alone.

  * step identity: score(slot, rb, re) equals, bit for bit, the pred a train step on the same rows leaves in the slot --
    for every model, gradient path and dense-layer precision, before and after updates (the bf16 weight copies refreshed);
  * accuracy: NFM fp32 scores against tests/ref64.py under the condition-scaled bound of test_kernel_shapes_gpu.py, bf16
    scores against the rounding-point emulation of test_mlp_bf16_gpu.py;
  * no side effects: parameters, optimizer state, dense layers and the following loss trajectory equal a twin context's
    that never scored;
  * blocks: NFM / Wide&Deep score a slot past 2 x 65536 rows in blocks, with the same bits as sub-range scores;
  * keyed slots, refusals and launch counts."""
import numpy as np
import pytest

import ref64
from test_kernel_shapes_gpu import _check_pctr
from test_mlp_bf16_gpu import _emulate

pytestmark = pytest.mark.gpu

F = 3000


def _batch(seed, rows, Fc=0, nnz_per=24, with_val=False, distinct=True):
    rng = np.random.RandomState(seed)
    cnt = rng.randint(nnz_per // 2, nnz_per + 1, size=rows)
    rp = np.zeros(rows + 1, np.int64)
    rp[1:] = np.cumsum(cnt)
    fid = (np.concatenate([rng.choice(F, c, replace=False) for c in cnt]) if distinct
           else rng.randint(0, F, int(rp[-1]))).astype(np.uint32)
    field = rng.randint(0, Fc, len(fid)).astype(np.uint16) if Fc else None
    val = (rng.rand(len(fid)) * 1.5 + 0.25).astype(np.float32) if with_val else None
    label = (rng.rand(rows) < 0.4).astype(np.int32)
    return rp, fid, field, val, label


# name: (model, k, Fc, deterministic, precision, hidden, env, masked, with_val)
def _cases(capi):
    FM, FFM, NFM, WND = capi.MODEL_FM, capi.MODEL_FFM, capi.MODEL_NFM, capi.MODEL_WND
    P32, P16 = capi.MLP_FP32, capi.MLP_BF16
    return {
        "fm_k16_compact": (FM, 16, 0, 0, P32, (), {}, False, False),
        "fm_k16_compact_val": (FM, 16, 0, 0, P32, (), {}, False, True),
        "fm_k10_dense": (FM, 10, 0, 0, P32, (), {}, False, True),
        "fm_det1": (FM, 16, 0, 1, P32, (), {}, False, False),
        "fm_det2": (FM, 16, 0, 2, P32, (), {}, False, False),
        "ffm_det0_warp": (FFM, 4, 8, 0, P32, (), {}, False, True),
        "ffm_det0_cta_k2": (FFM, 2, 8, 0, P32, (), {}, False, False),
        "ffm_det1": (FFM, 4, 8, 1, P32, (), {}, False, False),
        "ffm_det2": (FFM, 4, 8, 2, P32, (), {}, False, False),
        "nfm_fp32_det0": (NFM, 16, 0, 0, P32, (64, 32), {}, False, False),
        "nfm_fp32_det0_k10": (NFM, 10, 0, 0, P32, (64, 32), {}, False, False),
        "nfm_fp32_det1": (NFM, 16, 0, 1, P32, (64, 32), {}, False, False),
        "nfm_bf16_wgmma": (NFM, 16, 0, 0, P16, (128, 64), {}, False, False),
        "nfm_bf16_mma_masked": (NFM, 16, 0, 0, P16, (128, 64), {}, True, False),
        "nfm_bf16_mma_env": (NFM, 16, 0, 0, P16, (128, 64), {"LCTR_MLP_UMMA": "0"}, False, False),
        "wnd_fp32": (WND, 4, 8, 0, P32, (64, 32), {}, False, True),
        "wnd_bf16": (WND, 4, 8, 0, P16, (128, 64), {}, False, False),
    }


CASE_NAMES = ["fm_k16_compact", "fm_k16_compact_val", "fm_k10_dense", "fm_det1", "fm_det2", "ffm_det0_warp",
              "ffm_det0_cta_k2", "ffm_det1", "ffm_det2", "nfm_fp32_det0", "nfm_fp32_det0_k10", "nfm_fp32_det1",
              "nfm_bf16_wgmma", "nfm_bf16_mma_masked", "nfm_bf16_mma_env", "wnd_fp32", "wnd_bf16"]


def _params(capi, model, k, Fc, hidden, seed):
    rng = np.random.RandomState(seed)
    rowlen = k * (Fc if model == capi.MODEL_FFM else 1)
    W = (rng.randn(F) * 0.05).astype(np.float32)
    V = (rng.randn(F * rowlen) * 0.15).astype(np.float32)
    in0 = Fc * k if model == capi.MODEL_WND else k
    dims = [in0] + list(hidden) + [1]
    layers = [((rng.randn(dims[i + 1], dims[i]) * (1.5 / np.sqrt(dims[i]))).astype(np.float32),
               (rng.randn(dims[i + 1]) * 0.1).astype(np.float32)) for i in range(len(dims) - 1)]
    return W, V, layers, dims


def _make(capi, monkeypatch, name, rows, seed=1):
    model, k, Fc, det, prec, hidden, env, masked, with_val = _cases(capi)[name]
    for key, v in env.items():
        monkeypatch.setenv(key, v)  # read when the context prepares its dense layers
    c = capi.Context(model, F, k, field_cnt=Fc, hidden=hidden, mlp_precision=prec, deterministic=det, minibatch_size=rows)
    W, V, layers, dims = _params(capi, model, k, Fc, hidden, seed)
    c.upload_params(W, V)
    masks = []
    for l, (w, b) in enumerate(layers if hidden else []):
        c.mlp_upload(l, w, b)
        if l < len(hidden):
            m = np.ones(hidden[l], np.float32)
            if masked and l == 0:
                m[3] = 0.0
                c.mlp_set_mask(l, m)
            masks.append(m)
    rp, fid, field, val, label = _batch(seed + 100, rows, Fc if model in (capi.MODEL_FFM, capi.MODEL_WND) else 0,
                                        with_val=with_val)
    c.upload_batch(0, rp, fid, field, val, label)
    return c, dict(W=W, V=V, layers=layers, dims=dims, masks=masks, batch=(rp, fid, field, val, label), k=k, Fc=Fc)


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("name", CASE_NAMES)
def test_score_equals_the_train_steps_pred(name, monkeypatch):
    from lightctr_b200 import capi
    rows = 300
    c, _ = _make(capi, monkeypatch, name, rows)
    for rnd in range(2):
        s = c.score(0)
        c.train_step(0)
        assert np.array_equal(_bits(s), _bits(c.download_pred(0))), (name, rnd)
        for _ in range(3):  # updates: the next round scores refreshed parameters (and bf16 weight copies)
            c.train_step(0)
    c.close()


@pytest.mark.parametrize("name", ["fm_k16_compact", "fm_k10_dense", "ffm_det0_warp", "nfm_fp32_det0", "nfm_bf16_wgmma",
                                  "wnd_bf16"])
def test_score_of_a_sub_range_equals_the_step_on_it(name, monkeypatch):
    from lightctr_b200 import capi
    c, _ = _make(capi, monkeypatch, name, 300)
    c.train_step(0)
    rb, re = 37, 251
    s = c.score(0, rb, re)
    assert len(s) == re - rb
    c.train_step(0, rb, re)
    assert np.array_equal(_bits(s), _bits(c.download_pred(0)[rb:re]))
    assert len(c.score(0, 5, 5)) == 0
    c.close()


def _state(c, dims):
    """parameters, optimizer state, dense layers and dense gradients as the host sees them"""
    out = [*c.download_params(), *c.download_opt_state()]
    for l in range(len(dims) - 1 if len(dims) > 2 else 0):
        out += [*c.mlp_download(l, dims[l], dims[l + 1]), *c.mlp_download_grad(l, dims[l], dims[l + 1])]
    return out


def _scores(c, rows):
    c.score(0)
    c.score(0, 10, 200, download=False)
    c.score(0, 0, 0)
    c.score(0, rows - 1, rows)


@pytest.mark.parametrize("name", ["fm_k16_compact", "fm_k10_dense", "ffm_det0_warp", "ffm_det2", "nfm_fp32_det0",
                                  "nfm_bf16_wgmma", "nfm_bf16_mma_masked", "wnd_fp32", "wnd_bf16"])
def test_score_changes_no_state(name, monkeypatch):
    """on every path: what a train step leaves stays as it is through scores (the dense gradients stay zero)"""
    from lightctr_b200 import capi
    rows = 300
    c, info = _make(capi, monkeypatch, name, rows)
    c.train_step(0)
    before = _state(c, info["dims"])
    _scores(c, rows)
    after = _state(c, info["dims"])
    for x, y in zip(before, after):
        assert np.array_equal(_bits(x), _bits(y))
    if len(info["dims"]) > 2:
        assert not any(np.any(g) for l in range(len(info["dims"]) - 1)
                       for g in c.mlp_download_grad(l, info["dims"][l], info["dims"][l + 1]))
    c.close()


# the paths whose steps are bit-reproducible (no float REDs): a twin context that never scored follows the same trajectory
@pytest.mark.parametrize("name", ["fm_det1", "fm_det2", "nfm_fp32_det1"])
def test_steps_after_a_score_equal_a_twin_without_it(name, monkeypatch):
    from lightctr_b200 import capi
    rows = 300
    a, info = _make(capi, monkeypatch, name, rows)
    b, _ = _make(capi, monkeypatch, name, rows)
    for c in (a, b):
        c.train_step(0)
    _scores(a, rows)
    for step in range(3):
        la, lb = a.train_step(0), b.train_step(0)
        assert _bits(np.array(la)).tolist() == _bits(np.array(lb)).tolist(), (step, la, lb)
        assert np.array_equal(_bits(a.download_pred(0)), _bits(b.download_pred(0)))
    for x, y in zip(_state(a, info["dims"]), _state(b, info["dims"])):
        assert np.array_equal(_bits(x), _bits(y))
    a.close(); b.close()


@pytest.mark.parametrize("name", ["nfm_fp32_det0", "nfm_bf16_wgmma", "wnd_fp32"])
def test_blocks_of_a_large_slot(name, monkeypatch):
    """2 x 65536 + 123 rows: three dense blocks in one call, the same bits as sub-range calls and as the step"""
    from lightctr_b200 import capi
    model, k, Fc, det, prec, hidden, env, masked, with_val = _cases(capi)[name]
    rows = 2 * 65536 + 123
    c = capi.Context(model, F, k, field_cnt=Fc, hidden=hidden, mlp_precision=prec, minibatch_size=rows)
    W, V, layers, _ = _params(capi, model, k, Fc, hidden, 5)
    c.upload_params(W, V)
    for l, (w, b) in enumerate(layers):
        c.mlp_upload(l, w, b)
    c.upload_batch(0, *_batch(6, rows, Fc, nnz_per=6, distinct=False))
    whole = c.score(0)
    cuts = [0, 1000, 70001, 131072, rows]
    parts = np.concatenate([c.score(0, a, b) for a, b in zip(cuts[:-1], cuts[1:])])
    assert np.array_equal(_bits(whole), _bits(parts))
    c.train_step(0)
    assert np.array_equal(_bits(whole), _bits(c.download_pred(0)))
    c.close()


def test_nfm_fp32_score_vs_ref64(monkeypatch):
    from lightctr_b200 import capi
    c, info = _make(capi, monkeypatch, "nfm_fp32_det0", 300)
    s = c.score(0)
    rp, fid, _, val, label = info["batch"]
    z, wide, _, z_cond, wide_cond = ref64.nfm_forward(rp, fid, val, info["W"], info["V"], info["k"])
    p64, _, _, logit_cond = ref64.nfm_head(z, wide, info["layers"], capi.ACT_SIGMOID, None, label, z_cond, wide_cond)
    _check_pctr(s, p64, logit_cond)
    c.close()


@pytest.mark.parametrize("name", ["nfm_bf16_wgmma", "nfm_bf16_mma_masked"])
def test_nfm_bf16_score_vs_emulation(name, monkeypatch):
    torch = pytest.importorskip("torch")
    from lightctr_b200 import capi
    c, info = _make(capi, monkeypatch, name, 300)
    s = c.score(0)
    rp, fid, _, _, label = info["batch"]
    p_ref, _, _ = _emulate(torch, capi, rp, fid, label, info["W"], info["V"], info["k"], info["layers"], capi.ACT_SIGMOID,
                           info["masks"])
    assert np.max(np.abs(s - p_ref)) < 3e-3, np.max(np.abs(s - p_ref))  # bf16-ulp flips of single activations
    c.close()


def test_launch_counts(monkeypatch):
    from lightctr_b200 import capi
    for name, want in (("nfm_bf16_wgmma", 2), ("fm_k16_compact", 1), ("ffm_det0_warp", 1)):
        c, _ = _make(capi, monkeypatch, name, 300)
        n0 = c.launch_count()
        c.score(0)
        assert c.launch_count() - n0 == want, name
        c.close()


def _keyed_batch(seed, rows):
    from lightctr_b200.dist import fmix64
    rp, fid, _, _, label = _batch(seed, rows)
    return rp, fmix64(fid.astype(np.uint64) + np.uint64(11)), label


@pytest.mark.parametrize("model", ["fm", "nfm_bf16"])
def test_keyed_slots(model):
    from lightctr_b200 import capi
    from lightctr_b200.dist import fmix64
    k, rows, cap = 16, 400, 8000
    nfm = model == "nfm_bf16"
    kw = dict(hidden=(128, 64), mlp_precision=capi.MLP_BF16) if nfm else {}
    c = capi.Context(capi.MODEL_NFM if nfm else capi.MODEL_FM, cap, k, lr=0.01, key_mode=capi.KEYS_HASHED, **kw)
    c.set_key_init(0, 0.1)
    rp, keys, label = _keyed_batch(21, rows)
    c.upload_batch_keys(0, rp, keys, None, None, label)
    c.train_step(0)
    s = c.score(0)  # insert = 1: the step identity
    c.train_step(0)
    assert np.array_equal(_bits(s), _bits(c.download_pred(0)))
    # insert = 0: unseen keys sit on the null row, which scores as a zero row
    rng = np.random.default_rng(3)
    tkeys = keys.copy()
    unseen = rng.random(len(keys)) < 0.3
    tkeys[unseen] = fmix64(np.arange(unseen.sum(), dtype=np.uint64) + np.uint64(1 << 50))
    c.upload_batch_keys(1, rp, tkeys, None, None, label, insert=False)
    s1 = c.score(1)
    if not nfm:
        W, V = c.download_params()
        Wx, Vx = np.concatenate([W, [0.0]]).astype(np.float32), np.concatenate([V, np.zeros(k)]).astype(np.float32)
        rows_of = c.download_batch(1)[1]  # table rows; the null row is row `cap`
        assert np.all(rows_of[unseen] == cap)
        _, _, p64, _, logit_cond = ref64.fm_forward(rp, rows_of, None, Wx, Vx, k)
        _check_pctr(s1, p64, logit_cond)
    else:
        assert np.all(np.isfinite(s1)) and np.all((s1 > 0) & (s1 < 1))
    c.close()


def test_invalid_and_stale_slots_are_refused():
    from lightctr_b200 import capi
    k, rows = 8, 300
    rp, keys, label = _keyed_batch(31, rows)
    U = len(np.unique(keys))
    c = capi.Context(capi.MODEL_FM, U, k, key_mode=capi.KEYS_HASHED, key_evict=True)
    c.upload_batch_keys(0, rp, keys, None, None, label)
    c.train_step(0)
    keys2 = keys.copy()
    keys2[5] = np.uint64(123456789)  # no row left for it: the upload fails and leaves the slot unusable
    with pytest.raises(capi.LctrError, match="capacity"):
        c.upload_batch_keys(1, rp, keys2, None, None, label)
    with pytest.raises(capi.LctrError, match="no usable batch"):
        c.score(1)
    with pytest.raises(capi.LctrError, match="outside slot"):
        c.score(0, 0, rows + 1)
    c.evict_keys(max_rows=U // 2)
    with pytest.raises(capi.LctrError, match="stale"):
        c.score(0)
    c.close()
