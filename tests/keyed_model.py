"""numpy model of keyed contexts (csrc/keys.cu) shared by the keyed GPU tests: the lazy-init generator, the admission
sketch's cells, the upload clock and the eviction rule, and the sliding-window upload history they replay."""
import numpy as np

from lightctr_b200.dist import fmix64

GOLD = 0x9E3779B97F4A7C15
FC_FFM = 5  # fields of the FFM contexts of the eviction and tier tests
OPTS = {"adagrad": 0, "ftrl": 1, "ps_adagrad": 6}


def init_v(keys, rowlen, seed, scale):
    """the lazy-init generator of include/lightctr_b200.h / keys.cu: [len(keys), rowlen] float32"""
    hk = fmix64(keys)[:, None]
    j = np.arange(rowlen, dtype=np.uint64)[None, :]
    with np.errstate(over="ignore"):
        g = hk * np.uint64(rowlen) + j
        h = fmix64(g * np.uint64(GOLD) + np.uint64(seed))
    u1 = ((h & np.uint64(0x7fffff)).astype(np.float32) + np.float32(0.5)) * np.float32(2.0 ** -23)
    u2 = ((h >> np.uint64(24)) & np.uint64(0xffffff)).astype(np.float32) * np.float32(2.0 ** -24)
    r = np.sqrt(np.float32(-2.0) * np.log(u1))
    return (np.float32(scale) * r * np.cos(np.float32(6.2831853) * u2)).astype(np.float32)


def cells(keys, lw):
    """counter i of each key: fmix64(x ^ ((i + 1) * 0x9E3779B97F4A7C15)) >> (64 - log2_width), i = 0..3"""
    keys = np.asarray(keys, np.uint64)
    return [(fmix64(keys ^ np.uint64(((i + 1) * GOLD) % (1 << 64))) >> np.uint64(64 - lw)).astype(np.int64) for i in range(4)]


class Clock:
    """numpy model of the stamps: key -> clock of the insert-upload that last met it"""

    def __init__(self):
        self.clock, self.stamp = 0, {}

    def insert(self, keys):
        self.clock += 1
        for k in np.unique(keys).tolist():
            self.stamp[k] = self.clock

    def ages(self, table):
        return np.array([self.clock - self.stamp[k] for k in table.tolist()], np.int64)


def model_evict(table, ages, max_idle, max_rows):
    """evicted mask over the old rows and the renumbered row -> key map (include/lightctr_b200.h)"""
    ev = np.zeros(len(table), bool)
    if max_idle is not None:
        ev |= ages > max_idle
    if max_rows is not None and (~ev).sum() > max_rows:
        cut = np.sort(ages[~ev])[max_rows]  # a*: rows younger than the age of rank max_rows stay
        ev |= ages >= cut
    n_live = len(table) - int(ev.sum())
    holes = np.nonzero(ev[:n_live])[0]
    movers = n_live + np.nonzero(~ev[n_live:])[0]
    assert len(holes) == len(movers)
    new = table.copy()
    new[holes] = table[movers]
    return ev, new[:n_live]


class Batch:
    """rows of `per` keys; entry i has field i % FC_FFM"""

    def __init__(self, keys, per, rng):
        self.keys = np.ascontiguousarray(keys, np.uint64)
        rows = len(keys) // per
        self.rp = np.arange(0, rows * per + 1, per, dtype=np.int64)
        self.fld = (np.arange(len(keys)) % FC_FFM).astype(np.uint16)
        self.lab = (rng.random(rows) < 0.3).astype(np.int32)

    def upload(self, ctx, slot, insert=True):
        ctx.upload_batch_keys(slot, self.rp, self.keys, self.fld if ctx.Fc else None, None, self.lab, insert=insert)


def history(seed, n_up, universe=3000, rows=100, per=6):
    """n_up batches over a sliding window of the key universe: keys fall out of use as the window moves on"""
    rng = np.random.default_rng(seed)
    pool = fmix64(np.arange(universe, dtype=np.uint64) + np.uint64(1 << 33))
    out = []
    for i in range(n_up):
        lo = i * universe // (2 * n_up)
        out.append(Batch(pool[rng.integers(lo, lo + universe // 2, rows * per)], per, rng))
    return out


def replay(ctx, batches, clock=None, train=False):
    for i, b in enumerate(batches):
        b.upload(ctx, i % 8)
        if clock is not None:
            clock.insert(b.keys)
        if train:
            ctx.train_step(i % 8)


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def rows(ctx):
    """per-row arrays W [F], V [F, rowlen], s1W, s1V, s2W, s2V (s2 zero when the rule has none)"""
    F, r = ctx.F, ctx.rowlen
    W, V = ctx.download_params()
    s1, s2 = ctx.download_opt_state()
    return [W, V.reshape(F, r), s1[:F], s1[F:].reshape(F, r), s2[:F], s2[F:].reshape(F, r)]
