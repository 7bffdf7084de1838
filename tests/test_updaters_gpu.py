"""Every updater rule on every kernel that applies it, bit for bit against the oracle, on the exact batches of
tests/exact_batch.py (every gradient exact in fp32, so the only freedom left to a kernel is the update itself).

Each case runs three steps.  Each step starts from freshly uploaded dyadic parameters while the updater state stays on the
device, so step t + 1 starts from the state the kernel wrote; after each step W, V, s1 and s2 must equal the oracle's
expected step in every bit.  The batches hold hot ids (the compact updater's replica tile; a feature-major segment longer
than one task), ids met only in single-entry rows with a zero V row (an exactly zero V gradient, which every rule must
leave alone), FFM fields absent from a feature's rows and rows of 300 entries.  Ids name the applier instance, the shape
and the rule; minibatch_size alternates between 0 (the rows of the step) and 512."""
import numpy as np
import pytest

import exact_batch as eb

pytestmark = pytest.mark.gpu

F = 3000
FM, FFM = 1, 2

# (id, model, k, Fc, deterministic)
APPLIERS = [
    ("apply_compact_kernel-K4", FM, 4, 0, 0),
    ("apply_compact_kernel-K8", FM, 8, 0, 0),
    ("apply_compact_kernel-K16", FM, 16, 0, 0),
    ("apply_compact_kernel-K32", FM, 32, 0, 0),
    ("apply_kernel-VEC1-LPR4-fm_backward_kernel-K3", FM, 3, 0, 0),
    ("apply_kernel-VEC1-LPR8-fm_backward_kernel-K6", FM, 6, 0, 0),
    ("apply_kernel-VEC4-LPR4-fm_backward_kernel-K12", FM, 12, 0, 0),
    ("apply_kernel-VEC4-LPR8-fm_backward_kernel-K24", FM, 24, 0, 0),
    ("fm_backward_csc_kernel-LR4-K3", FM, 3, 0, 1),
    ("fm_backward_csc_kernel-LR8-K8", FM, 8, 0, 1),
    ("fm_backward_csc_kernel-LR32-K24", FM, 24, 0, 1),
    ("csc_apply_update-K8", FM, 8, 0, 2),
    ("csc_apply_update-K16", FM, 16, 0, 2),
    ("apply_kernel-VEC4-LPR4-SPL1-ffm_warp-Fc3-K4", FFM, 4, 3, 0),
    ("apply_kernel-VEC4-LPR32-SPL1-ffm_warp-Fc8-K16", FFM, 16, 8, 0),
    ("apply_kernel-VEC4-LPR32-SPL2-ffm_warp-Fc16-K16", FFM, 16, 16, 0),
    ("apply_kernel-VEC4-LPR32-SPL3-ffm_warp-Fc32-K12", FFM, 12, 32, 1),
    ("apply_kernel-VEC4-LPR32-SPL4-ffm_warp-Fc64-K8", FFM, 8, 64, 0),
    ("apply_kernel-VEC1-LPR16-ffm_fused_kernel-Fc5-K2", FFM, 2, 5, 0),
    ("apply_kernel-VEC1-LPR32-SPL3-ffm_fused_kernel-Fc13-K6", FFM, 6, 13, 1),
    ("ffm_backward_grouped_kernel-Fc4-K8", FFM, 8, 4, 2),
    ("ffm_backward_grouped_kernel-Fc16-K16", FFM, 16, 16, 2),
]

CASES = [pytest.param(a, rule, 0 if (i + j) % 2 == 0 else 512, id="%s-%s" % (a[0], rule))
         for i, a in enumerate(APPLIERS) for j, rule in enumerate(eb.RULES)]


def _same(what, got, want):
    bad = np.flatnonzero(got.view(np.uint32) != want.view(np.uint32))
    assert len(bad) == 0, "%s: %d of %d differ, first at %d: got %r, want %r" % (
        what, len(bad), len(got), bad[0], float(got[bad[0]]), float(want[bad[0]]))


def _context(rule, model, k, Fc, det, l2, mb, **kw):
    from lightctr_b200 import capi
    h = eb.HYPER
    return capi.Context(model, F, k, Fc, optimizer=eb.capi_opt(rule), lr=h["lr"], l2=l2, minibatch_size=mb,
                        momentum=h["beta1"], momentum_adam2=h["beta2"], ema_rate=h["ema"], deterministic=det, **kw)


def _check(ctx, rule, step, W, V, s1, s2):
    Wg, Vg = ctx.download_params()
    a, b = ctx.download_opt_state()
    _same("W step %d" % step, Wg, W)
    _same("V step %d" % step, Vg, V)
    _same("s1 step %d" % step, a, s1)
    if rule in eb.TWO_STATES:
        _same("s2 step %d" % step, b, s2)


def _steps(ctx, b, rule, seed, mb, s1, s2):
    """three steps, each from freshly uploaded parameters, the state left on the device; checked after each"""
    it = 0
    for step in range(3):
        W, V = eb.make_params(b, seed + 100 * step)
        gW, gV, _bits = eb.exact_grad(b, W, V)
        ctx.upload_params(W, V)
        ctx.train_step(0)
        W, V, s1, s2, it = eb.expected_step(rule, W, V, s1, s2, gW, gV, b.fid, mb or b.rows, eb.HYPER, it)
        _check(ctx, rule, step, W, V, s1, s2)


@pytest.mark.parametrize("applier,rule,mb", CASES)
def test_updater_bit_for_bit(applier, rule, mb):
    _name, model, k, Fc, det = applier
    seed = 1000 * k + 10 * Fc + det
    b = eb.make_batch(seed, F, k, Fc, scale=eb.SCALE[rule])
    s1, s2 = eb.make_state(b, rule, seed)
    ctx = _context(rule, model, k, Fc, det, b.l2, mb)
    ctx.upload_batch(0, b.rp, b.fid, b.fld if Fc else None, b.val, b.lab)
    ctx.upload_opt_state(s1, s2)
    _steps(ctx, b, rule, seed, mb, s1, s2)
    ctx.close()


@pytest.mark.parametrize("rule", ["ps_adagrad", "ps_dcasgda"])
def test_keyed_rows_start_at_the_server_state(rule):
    """keyed FM (compact updater): rows created on the device start at the server's state, s1 = 1e-7 (data_accum) and
    s2 = 0 (the shadow), then step as the dense context does, key by key (keys seeded in id order: row == id)"""
    from lightctr_b200 import capi, dist as ldist
    k, seed = 8, 4242
    b = eb.make_batch(seed, F, k, scale=eb.SCALE[rule])
    ctx = _context(rule, FM, k, 0, 0, b.l2, 0, key_mode=capi.KEYS_HASHED)
    keys = ldist.fmix64(np.arange(F))
    ctx.upload_keyed_params(keys, b.W, b.V)
    assert np.array_equal(ctx.lookup_keys(keys), np.arange(F))
    s1, s2 = ctx.download_opt_state()
    assert np.all(s1 == np.float32(1e-7)) and not s2.any()
    ctx.upload_batch_keys(0, b.rp, ldist.fmix64(b.fid), None, b.val, b.lab)
    _steps(ctx, b, rule, seed, 0, s1, s2)
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------
# streamed graphs: the compact updater and the device-grouped backward read OptParams from device memory (d_opt), staged
# per pipeline slot; 2 * LCTR_PIPE_DEPTH + 1 batches cycle every slot twice.  Each batch has features of its own, so its
# gradient is exact at the parameters uploaded once before the first batch.
# ------------------------------------------------------------------------------------------------------------------------
PIPE = 3  # LCTR_PIPE_DEPTH
STREAMED = [("apply_compact_kernel-K16-graph", 16, 0), ("csc_apply_update-K8-graph", 8, 2)]


@pytest.mark.parametrize("rule", eb.RULES)
@pytest.mark.parametrize("name,k,det", STREAMED, ids=[s[0] for s in STREAMED])
def test_streamed_updater_bit_for_bit(name, k, det, rule):
    n = 2 * PIPE + 1
    span = F // n
    seed = 77 + k
    batches = [eb.make_batch(seed + i, F, k, scale=eb.SCALE[rule], rows=280, id_base=i * span, id_span=span)
               for i in range(n)]
    W0, V0 = eb.make_params(batches[0], seed)
    for b in batches:
        V0.reshape(F, k)[b.single_only[::2]] = 0
    s1, s2 = eb.make_state(batches[0], rule, seed)
    ctx = _context(rule, FM, k, 0, det, batches[0].l2, 0)
    ctx.upload_params(W0, V0)
    ctx.upload_opt_state(s1, s2)
    tickets = []
    for i, b in enumerate(batches):
        if i >= PIPE:
            ctx.wait(tickets[i - PIPE])
        tickets.append(ctx.train_batch_async(b.rp, b.fid, None, b.val, b.lab))
    for t in tickets[-PIPE:]:
        ctx.wait(t)
    W, V, it = W0, V0, 0
    for b in batches:
        gW, gV, _bits = eb.exact_grad(b, W0, V0)  # its features still hold W0 / V0 when its step runs
        W, V, s1, s2, it = eb.expected_step(rule, W, V, s1, s2, gW, gV, b.fid, b.rows, eb.HYPER, it)
    _check(ctx, rule, n - 1, W, V, s1, s2)
    ctx.close()


# ------------------------------------------------------------------------------------------------------------------------
# two ranks on one GPU (tests/dist_updater_worker.py): the owner applies the sum of both ranks' records with the global
# minibatch.  Expected: the oracle's step on the union batch, minibatch = the global rows.
# ------------------------------------------------------------------------------------------------------------------------
DIST = [("push_rows_kernel-merge_apply_kernel-K8", 8), ("push_rows_kernel-merge_kernel-apply_kernel-VEC4-LPR4-K12", 12)]


@pytest.mark.parametrize("name,k", DIST, ids=[d[0] for d in DIST])
def test_two_ranks_updater_bit_for_bit(tmp_path, name, k):
    import dist_updater_worker as w
    import multirank as mr
    rows = 150
    mr.launch("dist_updater_worker.py", tmp_path, ["--k", str(k), "--rows", str(rows)])
    ranks = mr.load(tmp_path)
    own = np.arange(w.F) % 2
    own_s = np.concatenate([own, np.repeat(own, k)])
    for rule in eb.RULES:
        parts = [w.rank_batch(k, rows, rule, r) for r in range(2)]
        u = w.union(parts)
        s1, s2 = eb.make_state(parts[0], rule, 7)
        it = 0
        for step in range(w.STEPS):
            W, V = w.step_params(parts[0], step)
            gW, gV, _bits = eb.exact_grad(u, W, V)
            W, V, s1, s2, it = eb.expected_step(rule, W, V, s1, s2, gW, gV, u.fid, 2 * rows, eb.HYPER, it)
            got = {n: np.where((own_s if n[0] == "s" else own if n == "W" else np.repeat(own, k)) == 0,
                               ranks[0]["%s_%s%d" % (rule, n, step)], ranks[1]["%s_%s%d" % (rule, n, step)])
                   for n in ("W", "V", "s1", "s2")}
            _same("%s W step %d" % (rule, step), got["W"], W)
            _same("%s V step %d" % (rule, step), got["V"], V)
            _same("%s s1 step %d" % (rule, step), got["s1"], s1)
            if rule in eb.TWO_STATES:
                _same("%s s2 step %d" % (rule, step), got["s2"], s2)
