"""The weighted test-set metrics of lctr_eval_pred_weighted / lctr_eval_weighted restated in numpy (the rule is in
include/lightctr_b200.h), next to the unweighted metrics of lctr_eval / lctr_eval_pred they reduce to.

Both walk AucEvaluator's 2^24 - 1 buckets from the top over fp32 running totals.  numpy's add.accumulate is strictly
sequential, so the fp32 prefix sums of the walk are the device's chain, operation for operation; the logloss chain is a
row-order loop.  The logloss terms use numpy's logf / log, which may differ from the device's by an ulp per term."""
import numpy as np

HASH_LEN = (1 << 24) - 1


def buckets(pctr):
    """AucEvaluator's bucket of each pCTR: (p * (2^24 - 1)) in fp32, truncated"""
    idx = (np.asarray(pctr, np.float32) * np.float32(HASH_LEN)).astype(np.uint32)
    return np.minimum(idx, np.uint32(HASH_LEN))


def fixed_point(weight):
    """q_i = rint(w_i 2^(32-E)) with 2^(E-1) <= max w < 2^E; all zero when max w = 0"""
    w = np.asarray(weight, np.float32).astype(np.float64)
    M = float(w.max()) if len(w) else 0.0
    if M <= 0.0:
        return np.zeros(len(w), np.uint64)
    E = int(np.frexp(M)[1])
    return np.rint(np.ldexp(w, 32 - E)).astype(np.uint64)


def u64_to_f32(x):
    """fl32 of uint64 values, rounded once to nearest even as the device's conversion does (numpy's cast may round through
    float64 first)"""
    x = np.asarray(x, np.uint64)
    L = np.frexp(x.astype(np.float64))[1].astype(np.int64)  # bit length, or one more when the float64 rounded up to 2^L
    L = np.where((L > 0) & ((x >> np.maximum(L - 1, 0).astype(np.uint64)) == 0), L - 1, L)
    shift = np.maximum(L - 24, 0).astype(np.uint64)
    m = x >> shift
    rem = x - (m << shift)
    half = np.where(shift > 0, np.uint64(1) << np.maximum(shift, 1).astype(np.uint64) - np.uint64(1), np.uint64(0))
    up = (shift > 0) & ((rem > half) | ((rem == half) & ((m & np.uint64(1)) == 1)))
    m = m + up.astype(np.uint64)
    return np.ldexp(m.astype(np.float64), shift.astype(np.int64)).astype(np.float32)


def walk(pos, neg):
    """the fp32 trapezoid walk over per-bucket (positive, negative) sums, given in walk order (empty buckets add 0)"""
    keep = (pos | neg) != 0
    p = u64_to_f32(pos[keep])
    n = u64_to_f32(neg[keep])
    if len(p) == 0:
        return np.float32(0.0)
    tot_pos = np.add.accumulate(p, dtype=np.float32)
    tot_neg = np.add.accumulate(n, dtype=np.float32)
    prev_pos = np.concatenate([[np.float32(0)], tot_pos[:-1]]).astype(np.float32)
    prev_neg = np.concatenate([[np.float32(0)], tot_neg[:-1]]).astype(np.float32)
    dx = np.where(tot_neg > prev_neg, tot_neg - prev_neg, prev_neg - tot_neg).astype(np.float32)
    area = ((dx * (tot_pos + prev_pos).astype(np.float32)).astype(np.float32).astype(np.float64) / 2.0).astype(np.float32)
    auc = np.add.accumulate(area, dtype=np.float32)[-1]
    tp, tn = tot_pos[-1], tot_neg[-1]
    if not (tp > 0 and tn > 0):
        return np.float32(0.0)
    return np.float32(np.float32(auc / tp) / tn)


def _sums(pctr, label, amount):
    """per-bucket sums of `amount` (uint64) over label 1 and the other rows, in walk order (top bucket first)"""
    idx = buckets(pctr)
    pos_rows = np.asarray(label) == 1
    rev = (np.uint32(HASH_LEN) - idx).astype(np.int64)
    order = np.argsort(rev, kind="stable")
    r = rev[order]
    starts = np.flatnonzero(np.concatenate([[True], r[1:] != r[:-1]])) if len(r) else np.zeros(0, np.int64)
    a = np.asarray(amount, np.uint64)[order]
    pp = np.add.reduceat(np.where(pos_rows[order], a, np.uint64(0)), starts) if len(r) else np.zeros(0, np.uint64)
    nn = np.add.reduceat(np.where(pos_rows[order], np.uint64(0), a), starts) if len(r) else np.zeros(0, np.uint64)
    return pp.astype(np.uint64), nn.astype(np.uint64)


def _terms(pctr, label):
    p = np.asarray(pctr, np.float32)
    y = np.asarray(label).astype(np.float32)
    with np.errstate(divide="ignore"):
        t_pos = (-np.log(p)).astype(np.float64)
        t_neg = -np.log(1.0 - p.astype(np.float64))
    term = np.where(y == 1.0, t_pos, t_neg)
    ok = ((p > 0.5) & (y == 1.0)) | ((p < 0.5) & (y == 0.0))
    return term, ok


def _loss_chain(terms):
    loss = np.float32(0.0)
    with np.errstate(over="ignore"):  # weights near 3e38 overflow the fp32 chain to inf, as on the device
        for t in terms.tolist():
            loss = np.float32(float(loss) + t)
    return loss


def eval_unweighted(pctr, label):
    """lctr_eval_pred: (loss, correct, auc)"""
    term, ok = _terms(pctr, label)
    pos, neg = _sums(pctr, label, np.ones(len(term), np.uint64))
    return _loss_chain(term), int(ok.sum()), walk(pos, neg)


def eval_weighted(pctr, label, weight):
    """lctr_eval_pred_weighted: (loss, correct, auc), by the rule of the header"""
    w = np.asarray(weight, np.float32)
    term, ok = _terms(pctr, label)
    live = w != 0
    loss = _loss_chain(w[live].astype(np.float64) * term[live])
    cw = np.where(ok, w.astype(np.float64), 0.0)
    correct = float(np.add.accumulate(cw)[-1]) if len(cw) else 0.0
    pos, neg = _sums(pctr, label, fixed_point(w))
    return loss, correct, walk(pos, neg)
