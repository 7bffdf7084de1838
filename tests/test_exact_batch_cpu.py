"""The premises of tests/exact_batch.py, on the CPU: its batches are what it says they are, the oracle's sequential fp32
gradient on them equals ref64's float64 gradient bit for bit, and its expected updater step is the oracle trainers' own."""
import ctypes as C

import numpy as np
import pytest

import exact_batch as eb
from kernel_shapes_worker import make_batch as ordinary_batch, make_params as ordinary_params

SHAPES = [(8, 0), (32, 0), (3, 0), (4, 3), (16, 16), (8, 64), (6, 13)]  # (k, Fc)


def _ids(shapes):
    return ["FM-K%d" % k if not Fc else "FFM-Fc%d-K%d" % (Fc, k) for k, Fc in shapes]


@pytest.mark.parametrize("k,Fc", SHAPES, ids=_ids(SHAPES))
def test_generator_invariants(k, Fc):
    b = eb.make_batch(3, 3000, k, Fc, scale=15)
    x = b.x().astype(np.float64)
    assert set(np.unique(x / 2.0 ** 15)) <= {1.0, 2.0}
    assert np.all(b.W >= 20 * 2.0 ** -15) and np.all(b.V >= 0) and np.all(b.lab == 1)
    lens = np.diff(b.rp)
    assert lens.max() > 256 and np.sum(lens == 1) >= 20
    rows_of = np.repeat(np.arange(b.rows), lens)
    assert len(np.unique(rows_of[b.fid == b.hot[0]])) > 256  # the grouped backward splits this segment
    single = np.isin(b.fid, b.single_only)
    assert single.any() and np.all(lens[rows_of[single]] == 1)
    zero_rows = b.single_only[::2]
    assert np.isin(zero_rows, b.fid).any() and not b.V.reshape(b.F, -1)[zero_rows].any()
    gW, gV, bits = eb.exact_grad(b)
    assert eb.logits(b).min() >= eb.MIN_LOGIT and bits < eb.BUDGET_BITS
    gV = gV.reshape(b.F, -1)
    present = np.unique(b.fid)
    # batch features with an exactly zero V gradient (a zero V row in single-entry rows only) ...
    assert not gV[np.intersect1d(zero_rows, present)].any()
    assert np.all(gW[present] != 0)
    if Fc:  # ... and FFM fields absent from every row of a feature
        blocks = gV[present].reshape(len(present), Fc, k)
        assert np.any(~blocks.any(axis=2)) and np.any(blocks.any(axis=2))


@pytest.mark.parametrize("k,Fc", SHAPES, ids=_ids(SHAPES))
def test_oracle_gradient_equals_ref64_bit_for_bit(oracle_api, k, Fc):
    """orc_fm_pass / orc_ffm_pass sum in fp32 in the reference's order; on an exact batch that equals the float64 sum"""
    b = eb.make_batch(5, 3000, k, Fc, scale=eb.SCALE["adagrad"])
    gW, gV, _bits = eb.exact_grad(b)
    ds = oracle_api.Dataset(b.rp, b.fid, b.fld.astype(np.uint32), b.x(), b.lab, b.F, Fc)
    if Fc:
        o = oracle_api.FFMOracle(ds, k, b.W, b.V, l2=b.l2)
    else:
        o = oracle_api.FMOracle(ds, k, b.W, b.V, l2=b.l2)
    o.forward_backward()
    assert np.all(o.pred == np.float32(1.0 + eb.D))
    assert np.array_equal(o.update_g.view(np.uint32), np.concatenate([gW, gV]).view(np.uint32))


def _ordinary(oracle_api, k, Fc, seed):
    rp, fid, fld, val, lab = ordinary_batch(seed, 2000, rows=120, Fc=Fc, with_val=True)
    ds = oracle_api.Dataset(rp, fid, fld.astype(np.uint32), val, lab, 2000, Fc)
    W, V = ordinary_params(seed, 2000, k, Fc)
    V.reshape(2000, -1)[fid[np.diff(rp)[np.repeat(np.arange(len(lab)), np.diff(rp))] == 1]] = 0  # zero V gradients
    return ds, W, V


@pytest.mark.parametrize("rule", eb.RULES)
def test_expected_step_is_the_fm_oracle_step(oracle_api, rule):
    """expected_step on FMOracle's own gradient (an ordinary batch, random state) moves W, V and both states exactly as
    FMOracle.apply does, over two steps (Adam's counter carried)"""
    k = 5
    ds, W, V = _ordinary(oracle_api, k, 0, 21)
    o = oracle_api.FMOracle(ds, k, W, V)
    o.opt = rule
    n = ds.feature_cnt * (k + 1)
    rng = np.random.default_rng(1)
    o.accum = (rng.random(n) * 1e-3).astype(np.float32)
    o.s2 = (rng.random(n) * 1e-3).astype(np.float32)
    o.iter = C.c_size_t(0)
    o._ps_init = True
    s1, s2, it = o.accum.copy(), o.s2.copy(), 0
    for _ in range(2):
        o.forward_backward()
        g = o.update_g.copy()
        W0, V0 = o.W.copy(), o.V.copy()
        o.apply()
        W1, V1, s1, s2, it = eb.expected_step(rule, W0, V0, s1, s2, g[:ds.feature_cnt], g[ds.feature_cnt:], ds.fid,
                                              ds.rows, eb.HYPER, it)
        for got, want in ((W1, o.W), (V1, o.V), (s1, o.accum)):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        if rule in eb.TWO_STATES:
            assert np.array_equal(s2.view(np.uint32), o.s2.view(np.uint32))
        assert it == o.iter.value
    assert not np.array_equal(W1, W) and not np.array_equal(V1, V)


@pytest.mark.parametrize("rule", [r for r in eb.RULES if r not in eb.PS_RULES])
def test_expected_step_is_the_ffm_oracle_step(oracle_api, rule):
    k, Fc = 3, 4
    ds, W, V = _ordinary(oracle_api, k, Fc, 31)
    o = oracle_api.FFMOracle(ds, k, W, V, optimizer=rule)
    rng = np.random.default_rng(2)
    o.s1[:] = rng.random(len(o.s1)) * 1e-3
    o.s2[:] = rng.random(len(o.s2)) * 1e-3
    s1, s2, it = o.s1.copy(), o.s2.copy(), 0
    for _ in range(2):
        o.forward_backward()
        g = o.update_g.copy()
        W0, V0 = o.W.copy(), o.V.copy()
        o.apply()
        W1, V1, s1, s2, it = eb.expected_step(rule, W0, V0, s1, s2, g[:ds.feature_cnt], g[ds.feature_cnt:], ds.fid,
                                              ds.rows, eb.HYPER, it)
        for got, want in ((W1, o.W), (V1, o.V), (s1, o.s1)):
            assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
        if rule in eb.TWO_STATES:
            assert np.array_equal(s2.view(np.uint32), o.s2.view(np.uint32))
        assert it == o.iter.value


def test_zero_gradient_leaves_parameter_server_state_alone(oracle_api):
    """the parameter-server rules skip a zero gradient: DCASGD keeps its shadow, DCASGDA its accumulator"""
    F, k = 4, 2
    W = np.full(F, 0.5, np.float32)
    V = np.full(F * k, 0.25, np.float32)
    s1 = np.full(F * (k + 1), 0.01, np.float32)
    s2 = np.full(F * (k + 1), 0.125, np.float32)
    gW = np.array([0.5, 0, 0, 0], np.float32)
    gV = np.zeros(F * k, np.float32)
    for rule in ("ps_dcasgd", "ps_dcasgda"):
        W1, V1, a, b, _ = eb.expected_step(rule, W, V, s1, s2, gW, gV, [0, 1], 10, eb.HYPER, 0)
        assert W1[0] != W[0] and np.array_equal(W1[1:], W[1:]) and np.array_equal(V1, V)
        assert b[0] != s2[0] and np.array_equal(b[1:], s2[1:])
        if rule == "ps_dcasgda":
            assert a[0] != s1[0] and np.array_equal(a[1:], s1[1:])
