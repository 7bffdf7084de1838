"""Batches whose FM / FFM gradients are exact in fp32, and the updater step the oracle takes on them.

Every row's logit is >= 20, so the sigmoid saturates at exactly 0.99999988f and, with label 1, every kernel computes
d = p - y = -2^-23 exactly.  Values x are small powers of two, W >= 0 and V >= 0 are dyadic with few significant bits and
l2 is a power of two, so every per-entry gradient term is a multiple of one quantum Q.  While the sum of |terms| of a
coordinate stays below 2^20 Q (`exact_grad`, from tests/ref64.py's condition figures), every partial sum is exact in fp32:
any summation order, with or without FMA, in fp32 or in double, gives the same bits.  The gradient of a kernel therefore
equals ref64's float64 gradient exactly, and so does the update it applies: `expected_step` runs the oracle's pinned
per-array updaters on that gradient, and a test compares parameters and updater state bit for bit.

A scale s multiplies x by 2^s, divides W and V by 2^s and multiplies l2 by 2^2s: the logits stay put and every gradient
scales by 2^s, which puts |g / minibatch| where a rule's constants (the 1e-7 epsilons, FTRL's alpha, beta and lambda1)
matter."""
import ctypes as C

import numpy as np

import ref64

RULES = ["adagrad", "ftrl", "adam", "rmsprop", "adadelta", "ps_sgd", "ps_adagrad", "ps_dcasgd", "ps_dcasgda"]
PS_RULES = ("ps_sgd", "ps_adagrad", "ps_dcasgd", "ps_dcasgda")
TWO_STATES = ("ftrl", "adam", "adadelta", "ps_dcasgd", "ps_dcasgda")
D = -2.0 ** -23        # p - y of every row: float(0.99999988f) - 1
MIN_LOGIT = 20.0
BUDGET_BITS = 20

# per rule: the scale s (gradient x 2^s) that puts |g / minibatch| (|g| for FTRL) where the rule's constants act
SCALE = dict(adagrad=15, ftrl=15, adam=4, rmsprop=16, adadelta=14, ps_sgd=15, ps_adagrad=14, ps_dcasgd=17, ps_dcasgda=19)
HYPER = dict(lr=0.05, beta1=0.8, beta2=0.999, ema=0.99)


def capi_opt(rule):
    from lightctr_b200 import capi
    return getattr(capi, "OPT_" + rule.upper())


class Batch:
    """CSR batch (labels all 1) with its dyadic parameters.  fid, fld (uint16), val (None = all ones), F, k, Fc (0 = FM),
    scale, l2; W, V; single_only (ids that occur in single-entry rows only), hot (ids in most rows)."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    @property
    def rows(self):
        return len(self.rp) - 1

    @property
    def rowlen(self):
        return self.k * max(self.Fc, 1)

    def x(self):
        return np.ones(len(self.fid), np.float32) if self.val is None else self.val


def make_batch(seed, F, k, Fc=0, rows=300, scale=0, n_hot=2, long_row=300, max_len=16, with_val=True, id_base=0,
               id_span=None):
    """rows of 1..max_len entries, a few single-entry rows, one row of `long_row` entries, and hot ids 0..n_hot-1 (+ id_base)
    in all but a few rows (hot id 0 is in more than 256 rows when rows > 270, so the grouped backward splits its segment);
    ids id_base + n_hot + [0, 20) occur only in single-entry rows, half of them with an all-zero V row (their V gradient
    is exactly zero).  Features come from [id_base, id_base + id_span).  FFM: each row draws its fields from a few of the
    Fc fields, so many (feature, field) pairs are absent from the batch.  Values in {1, 2} * 2^scale; with_val=False
    (scale 0 only) leaves them out, x = 1."""
    rng = np.random.default_rng(seed)
    span = id_span or F - id_base
    n_single = 20
    single = np.arange(n_hot, n_hot + n_single) + id_base
    pool = np.arange(n_hot + n_single, span) + id_base
    lens = rng.integers(2, max_len + 1, rows)
    single_rows = rng.choice(rows, 24, replace=False)
    lens[single_rows] = 1
    lens[rng.choice(np.setdiff1d(np.arange(rows), single_rows))] = long_row
    fid, fld = [], []
    for r, n in enumerate(lens):
        if n == 1:
            ids = np.array([single[r % n_single] if r % 3 else rng.choice(pool)])
        else:
            ids = rng.choice(pool, n, replace=False)
            if rng.random() < 0.99:
                ids[0] = id_base
            if n_hot > 1 and n >= 3 and rng.random() < 0.5:
                ids[1] = id_base + 1 + rng.integers(0, n_hot - 1)
        fid.append(ids)
        if Fc:
            few = rng.choice(Fc, min(Fc, 3), replace=False)
            fld.append(rng.choice(few, len(ids)))
        else:
            fld.append(np.zeros(len(ids), np.int64))
    rp = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    fid = np.concatenate(fid).astype(np.uint32)
    fld = np.concatenate(fld).astype(np.uint16)
    if with_val:
        val = (rng.integers(1, 3, len(fid)) * 2.0 ** scale).astype(np.float32)
    else:
        assert scale == 0, "a batch without values has x = 1: scale it with values"
        val = None
    b = Batch(rp=rp, fid=fid, fld=fld, val=val, lab=np.ones(rows, np.int32), F=F, k=k, Fc=Fc, scale=scale,
              l2=float(2.0 ** (-23 + 2 * scale)), single_only=single, hot=np.arange(n_hot) + id_base)
    b.W, b.V = make_params(b, seed)
    return b


def make_params(b, seed):
    """W in [20, 31] * 2^-s (every logit >= 20 with x >= 2^s), V in {0, 1/4, 1/2, 3/4} * 2^-s, the V rows of half the
    single-entry-only ids zero"""
    rng = np.random.default_rng(seed + 7)
    s = 2.0 ** -b.scale
    W = (rng.integers(20, 32, b.F) * s).astype(np.float32)
    V = (rng.integers(0, 4, (b.F, b.rowlen)) * 0.25 * s).astype(np.float32)
    V[b.single_only[::2]] = 0
    return W, V.reshape(-1)


def make_state(b, rule, seed):
    """nonzero starting state (s1, s2) of F * (rowlen + 1) floats, W part first, at the scale of the batch's gradients:
    FTRL z near +-lambda1, Adam m of both signs, the DCASGD shadow close to but not equal to w"""
    rng = np.random.default_rng(seed + 11)
    n = b.F * (b.rowlen + 1)
    g1 = 2.0 ** (b.scale - 23) * 40 / b.rows  # a typical |g / minibatch|
    s1 = np.zeros(n, np.float32)
    s2 = np.zeros(n, np.float32)
    u = rng.random(n)
    if rule in ("adagrad", "rmsprop", "adadelta"):
        s1[:] = u * g1 * g1
        if rule == "adadelta":
            s2[:] = rng.random(n) * g1 * g1
    elif rule == "ftrl":
        s1[:] = np.where(u < 0.5, -1, 1) * (0.9 + 0.2 * rng.random(n))
        s2[:] = rng.random(n) * 4
    elif rule == "adam":
        s1[:] = (u - 0.5) * g1
        s2[:] = rng.random(n) * g1 * g1
    elif rule in ("ps_adagrad", "ps_dcasgda"):
        s1[:] = np.float32(1e-7) + u * g1 * g1
    if rule in ("ps_dcasgd", "ps_dcasgda"):
        w = np.concatenate([b.W, b.V])
        s2[:] = w * (1 + (rng.random(n) - 0.5) * 2.0 ** -8)
    return s1, s2


def logits(b, W=None, V=None):
    W, V = (b.W, b.V) if W is None else (W, V)
    if b.Fc:
        return ref64.ffm_forward(b.rp, b.fid, b.fld, b.val, W, V, b.Fc, b.k)[0]
    return ref64.fm_forward(b.rp, b.fid, b.val, W, V, b.k)[1]


def grad64(b, W=None, V=None):
    """(gW [F], gV [F * rowlen], gW_cond, gV_cond) in float64 at p = 0.99999988 on every row"""
    W, V = (b.W, b.V) if W is None else (W, V)
    pred = np.full(b.rows, 1.0 + D)
    if b.Fc:
        gW, gV, cW, cV = ref64.ffm_grad(b.rp, b.fid, b.fld, b.val, b.lab, W, V, b.Fc, b.k, pred, b.l2)
    else:
        sumvx = ref64.fm_forward(b.rp, b.fid, b.val, W, V, b.k)[0]
        gW, gV, cW, cV = ref64.fm_grad(b.rp, b.fid, b.val, b.lab, W, V, b.k, pred, sumvx, b.l2)
    return gW, gV.reshape(-1), cW, cV.reshape(-1)


def lowbit(a):
    """the smallest lowest-set-bit value over the nonzero entries of a (float64, every entry dyadic)"""
    a = np.abs(np.asarray(a, np.float64).ravel())
    a = a[a != 0]
    m, e = np.frexp(a)
    n = (m * 2.0 ** 53).astype(np.int64)
    return float(np.min((n & -n).astype(np.float64) * np.ldexp(1.0, e - 53)))


def quantum(b, W=None, V=None):
    """Q dividing every per-entry gradient term: d x, l2 w (gW); (sumVX - x v) * gradW, l2 v (FM gV); d x_i x_j v, l2 v
    (FFM gV).  The lowest set bit of a product of dyadics is the product of theirs."""
    W, V = (b.W, b.V) if W is None else (W, V)
    lx, lv, lw, ld, l2 = lowbit(b.x()), lowbit(V), lowbit(W), abs(D), b.l2
    qW = min(ld * lx, l2 * lw)
    qV = min(lx * lv * qW, l2 * lv) if not b.Fc else min(ld * lx * lx * lv, l2 * lv)
    return min(qW, qV)


def exact_grad(b, W=None, V=None):
    """the batch's gradient as every kernel holds it (float32), after checking the premises: every float64 logit
    >= MIN_LOGIT and log2(max(cond) / Q) < BUDGET_BITS, under which every summation order of every coordinate is exact
    in fp32 (so the cast from float64 is exact too).  Returns (gW, gV, bits)."""
    W, V = (b.W, b.V) if W is None else (W, V)
    z = logits(b, W, V)
    assert z.min() >= MIN_LOGIT, ("logit", float(z.min()))
    gW, gV, cW, cV = grad64(b, W, V)
    bits = float(np.log2(max(cW.max(), cV.max()) / quantum(b, W, V)))
    assert bits < BUDGET_BITS, ("budget", bits)
    g32W, g32V = gW.astype(np.float32), gV.astype(np.float32)
    assert np.array_equal(g32W.astype(np.float64), gW) and np.array_equal(g32V.astype(np.float64), gV)
    return g32W, g32V, bits


def expected_step(rule, W, V, s1, s2, gW, gV, batch_ids, minibatch, hyper, adam_iter):
    """One updater step of the oracle in the reference order: the W call, then the V call (Adam's counter advances with
    each call).  W [F], V [F * rowlen], s1 / s2 [F * (rowlen + 1)] (W part first), gW / gV the batch gradient.  The five
    trainer rules sweep every coordinate and skip the zero gradients; the parameter-server rules update the coordinates
    of the batch's features whose gradient is nonzero (the worker pushes no zero gradient, push.h:62-65), as
    FMOracle.apply does.  Returns (W, V, s1, s2, adam_iter), new arrays."""
    from oracle import api
    L = api.lib()
    F = len(W)
    rowlen = len(V) // F
    W, V, s1, s2 = (np.array(a, np.float32) for a in (W, V, s1, s2))
    lr = np.float32(hyper["lr"])
    it = C.c_size_t(adam_iter)
    ids = np.unique(np.asarray(batch_ids, np.int64))
    for w, g, lo, hi in ((W, gW, 0, F), (V, gV, F, F + F * rowlen)):
        g = np.array(g, np.float32)
        a, b = s1[lo:hi], s2[lo:hi]  # views
        if rule == "adagrad":
            L.orc_adagrad(hi - lo, w, g, a, minibatch, lr)
        elif rule == "ftrl":
            L.orc_ftrl(hi - lo, w, g, a, b, 1)
        elif rule == "adam":
            L.orc_adam(hi - lo, w, g, a, b, C.byref(it), minibatch, lr, np.float32(hyper["beta1"]),
                       np.float32(hyper["beta2"]))
        elif rule == "rmsprop":
            L.orc_rmsprop(hi - lo, w, g, a, minibatch, lr, np.float32(hyper["ema"]))
        elif rule == "adadelta":
            L.orc_adadelta(hi - lo, w, g, a, b, minibatch, np.float32(hyper["beta1"]))
        else:
            kind = PS_RULES.index(rule)
            idx = ids if lo == 0 else (ids[:, None] * rowlen + np.arange(rowlen)[None, :]).ravel()
            idx = idx[g[idx] != 0]
            ww, gg, aa, sh = w[idx].copy(), g[idx].copy(), a[idx].copy(), b[idx].copy()
            L.orc_ps_update(kind, len(idx), ww, gg, aa, sh, minibatch, lr, 0)
            w[idx], a[idx] = ww, aa
            if kind >= 2:
                b[idx] = sh
    if rule not in TWO_STATES:
        s2[:] = 0
    return W, V, s1, s2, it.value
