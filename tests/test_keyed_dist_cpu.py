"""Keyed mode on several GPUs, host side: the owner rule (top bits of fmix64), its balance, the merge of per-rank keyed
shards, and the unchanged lctr_cfg layout (the sharded keyed table needs no new cfg field)."""
import ctypes as C
import math
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M64 = (1 << 64) - 1


def _fmix64_py(k):
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & M64
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & M64
    k ^= k >> 33
    return k


def test_owner_of_key_is_top_bits_of_fmix64():
    from lightctr_b200 import dist as ldist
    rng = np.random.default_rng(3)
    keys = np.concatenate([rng.integers(0, 1 << 63, 500, dtype=np.int64).astype(np.uint64) * np.uint64(2) + np.uint64(1),
                           np.arange(50, dtype=np.uint64), np.array([M64 - 1], np.uint64)])
    for world in (1, 2, 4, 8):
        got = ldist.owner_of_key(keys, world)
        shift = world.bit_length() - 1
        want = [(_fmix64_py(int(k)) >> (64 - shift)) if shift else 0 for k in keys.tolist()]
        assert got.tolist() == want
        assert np.all((got >= 0) & (got < world))
    assert [int(x) for x in ldist.fmix64(keys[:20])] == [_fmix64_py(int(k)) for k in keys[:20].tolist()]


def test_shards_balanced_on_a_million_keys():
    """the owner of fmix64(key) is uniform: every shard's count within 6 binomial standard deviations of n / world"""
    from lightctr_b200 import dist as ldist
    n = 10 ** 6
    keys = ldist.fmix64(np.arange(n, dtype=np.uint64))  # hashed ids, as a Criteo pipeline would feed them
    for world in (2, 4, 8):
        cnt = np.bincount(ldist.owner_of_key(keys, world), minlength=world)
        p = 1.0 / world
        assert cnt.sum() == n
        assert np.all(np.abs(cnt - n * p) <= 6 * math.sqrt(n * p * (1 - p))), cnt


def test_merge_keyed_shards():
    from lightctr_b200 import dist as ldist
    world, cap, rowlen = 2, 6, 3
    keys = [np.array([11, 13, 17], np.uint64), np.array([19, 23], np.uint64)]
    W, V = [], []
    for r in range(world):
        w = np.full(cap, np.nan, np.float32)
        v = np.full((cap, rowlen), np.nan, np.float32)
        for l in range(len(keys[r])):
            g = l * world + r
            w[g] = 100 * r + l
            v[g] = np.arange(rowlen) + 10 * (100 * r + l)
        W.append(w)
        V.append(v.reshape(-1))
    m = ldist.merge_keyed_shards(keys, W, V, world)
    assert sorted(m) == [11, 13, 17, 19, 23]
    assert m[17][0] == 2 and np.array_equal(m[17][1], np.arange(rowlen) + 20)
    assert m[23][0] == 101 and np.array_equal(m[23][1], np.arange(rowlen) + 1010)


def test_cfg_layout_unchanged():
    """lctr_cfg keeps the size and offsets it had with keyed mode single-GPU only"""
    from lightctr_b200 import capi
    src = ('#include "lightctr_b200.h"\n#include <stdio.h>\n#include <stddef.h>\n'
           'int main(){printf("%zu %zu %zu %zu %zu\\n", sizeof(lctr_cfg), offsetof(lctr_cfg, rank), '
           'offsetof(lctr_cfg, key_mode), offsetof(lctr_cfg, key_evict), offsetof(lctr_cfg, reserved));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.c")
        open(p, "w").write(src)
        subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), p, "-o", os.path.join(d, "s")])
        size, off_rank, off_mode, off_evict, off_res = map(int, subprocess.check_output([os.path.join(d, "s")]).split())
    assert size == C.sizeof(capi.Cfg) == 176
    assert (off_rank, off_mode, off_evict, off_res) == (capi.Cfg.rank.offset, capi.Cfg.key_mode.offset,
                                                        capi.Cfg.key_evict.offset, capi.Cfg.reserved.offset)
