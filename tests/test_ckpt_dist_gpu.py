"""Checkpoints of sharded trainers (csrc/checkpoint.cu): 2 ranks sharing cuda:0 over CUDA IPC save per-rank shard files,
resume from them, and reshard them onto one GPU; a single-GPU file is resharded onto 2 ranks; the refused loads leave the
context as it was."""
import os

import numpy as np
import pytest

import dist_ckpt_worker as wk
import multirank as mr

pytestmark = pytest.mark.gpu


def _run(tmp_path, extra):
    mr.launch("dist_ckpt_worker.py", tmp_path, extra)


def _args(**kw):
    import argparse
    base = dict(model="fm", opt=0, keyed=False, F=20000, k=16, rows=256)
    base.update(kw)
    return argparse.Namespace(**base)


def _cli(a):
    return ["--model", a.model, "--opt", str(a.opt), "--F", str(a.F), "--k", str(a.k), "--rows", str(a.rows)] + \
        (["--keyed"] if a.keyed else [])


def _merge_pair(parts, F):
    """global [W part | V part] arrays (opt state) of 2 ranks, each valid at the rows it owns"""
    from lightctr_b200 import dist as ldist
    w = ldist.merge_shards([p[:F] for p in parts], 2, F)
    v = ldist.merge_shards([p[F:] for p in parts], 2, F)
    return np.concatenate([w, v])


def _merged(parts, prefix, F):
    from lightctr_b200 import dist as ldist
    out = {x: ldist.merge_shards([p[prefix + x] for p in parts], 2, F) for x in ("W", "V")}
    for x in ("s1", "s2"):
        out[x] = _merge_pair([p[prefix + x] for p in parts], F)
    return out


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _keyed_rows(keys, W, V, S1, S2, F, rowlen):
    """key -> (W, V row, s1 row, s2 row) of a 2-rank keyed save, from the ranks' global downloads"""
    out = {}
    for r in range(2):
        g = np.arange(len(keys[r])) * 2 + r
        for key, gg in zip(keys[r].tolist(), g):
            out[key] = (W[gg], V[gg * rowlen:(gg + 1) * rowlen], S1[gg], S1[F + gg * rowlen:F + (gg + 1) * rowlen],
                        S2[gg], S2[F + gg * rowlen:F + (gg + 1) * rowlen])
    return out


CASES = {
    "fm_adagrad": _args(),
    "ffm_ftrl": _args(model="ffm", opt=1, F=6000, k=4, rows=128),
    "nfm_adam": _args(model="nfm", opt=2, F=8000, k=16, rows=128),
    "keyed_fm": _args(keyed=True),
}


@pytest.mark.parametrize("case", list(CASES))
def test_resume_and_reshard_to_one_gpu(tmp_path, case):
    """3 steps + save_sharded + fresh contexts (create, connect, load_sharded, upload again) + 3 steps against 6 steps in
    one go; then the final save of the 2 ranks loaded into one world-1 context."""
    from lightctr_b200 import dist as ldist
    a = CASES[case]
    _run(tmp_path, ["--mode", "resume"] + _cli(a))
    parts = mr.load(tmp_path)
    rowlen = a.k * (39 if a.model == "ffm" else 1)
    F = mr.CAP_MULT * a.F if a.keyed else a.F
    # the save -> load round trip itself is exact: every download equal bit for bit
    assert all(bool(p["round_trip"]) for p in parts)
    # the continuation: deterministic = 0 (the only mode on several GPUs) sums gradients with REDs in arbitrary order, so
    # two runs of the same steps agree to rounding, not bit for bit
    sa, sb = parts[0]["stats_a"], parts[0]["stats_b"]
    assert np.allclose(sa[:, 0], sb[:, 0], rtol=1e-6, atol=0) and np.array_equal(sa[:, 1], sb[:, 1]), (sa, sb)
    # (the FTRL accumulators z and n amplify those rounding differences most)
    ma, mb = _merged(parts, "a_", F), _merged(parts, "b_", F)
    tol = {"W": 1e-5, "V": 1e-5, "s1": 1e-4, "s2": 1e-4}
    if not a.keyed:
        for x in ma:
            assert np.allclose(ma[x], mb[x], rtol=tol[x], atol=tol[x]), (x, float(np.max(np.abs(ma[x] - mb[x]))))
    else:  # a keyed upload numbers a batch's new keys in arbitrary order, so the runs compare key by key
        for r, p in enumerate(parts):
            assert set(p["a_keys"].tolist()) == set(p["b_keys"].tolist())
            assert np.all(ldist.owner_of_key(p["b_keys"], 2) == r)
        ka = _keyed_rows([p["a_keys"] for p in parts], ma["W"], ma["V"], ma["s1"], ma["s2"], F, rowlen)
        kb = _keyed_rows([p["b_keys"] for p in parts], mb["W"], mb["V"], mb["s1"], mb["s2"], F, rowlen)
        for key, va in ka.items():
            for x, y, t in zip(va, kb[key], (1e-5, 1e-5, 1e-4, 1e-4, 1e-4, 1e-4)):
                assert np.allclose(x, y, rtol=t, atol=t), key
    dims = mr.layer_dims(a.model, a.k)
    for l in range(len(dims) - 1):
        for r in range(2):
            assert np.allclose(parts[r]["a_mlp_w%d" % l], parts[r]["b_mlp_w%d" % l], rtol=1e-5, atol=1e-6)

    # reshard 2 -> 1: the final save into one GPU
    final = os.path.join(str(tmp_path), "final")
    paths, world = ldist.find_shards(final)
    assert world == 2
    c = wk.context(a, 0, 1)
    c.load_checkpoint_shards(paths)
    W, V = c.download_params()
    s1, s2 = c.download_opt_state()
    path1 = os.path.join(str(tmp_path), "one")
    c.save_checkpoint(path1)
    step1 = ldist.checkpoint_info(path1)[:2]
    assert step1 == ldist.checkpoint_info(paths[0])[:2] == ldist.checkpoint_info(paths[1])[:2]
    assert step1[0] == 2 * wk.HALF and (step1[1] > 0) == (a.opt == 2)
    for l in range(len(dims) - 1):
        w, b = c.mlp_download(l, dims[l], dims[l + 1])
        assert np.array_equal(_bits(w), _bits(parts[0]["b_mlp_w%d" % l])) and np.array_equal(_bits(b), _bits(parts[0]["b_mlp_b%d" % l]))
    if not a.keyed:
        mb = _merged(parts, "b_", F)
        for x, got in (("W", W), ("V", V), ("s1", s1)) + ((("s2", s2),) if a.opt else ()):
            assert np.array_equal(_bits(got), _bits(mb[x])), x
    else:
        keys = [p["b_keys"] for p in parts]
        mb = _merged(parts, "b_", F)
        ref = _keyed_rows(keys, mb["W"], mb["V"], mb["s1"], mb["s2"], F, rowlen)
        got_keys = c.download_keys()
        assert np.array_equal(got_keys, np.concatenate(keys))  # source order: rank 0's rows, then rank 1's
        for i, key in enumerate(got_keys.tolist()):
            w, v, a1w, a1v, _, _ = ref[key]
            assert _bits(np.float32(W[i])) == _bits(np.float32(w))
            assert np.array_equal(_bits(V[i * rowlen:(i + 1) * rowlen]), _bits(v))
            assert _bits(np.float32(s1[i])) == _bits(np.float32(a1w))
            assert np.array_equal(_bits(s1[F + i * rowlen:F + (i + 1) * rowlen]), _bits(a1v))
        n = len(got_keys)
        assert not np.any(W[n:]) and not np.any(V[n * rowlen:])  # rows past the keys as lctr_create leaves them
    c.close()


def _single_file(tmp_path, a, name, steps=3):
    """a single-GPU checkpoint of `a`'s world-1 context after `steps` steps on the global batches of 2 ranks"""
    per_rank = [mr.train_batches(a.F, a.rows, steps, r) for r in range(2)]
    c = wk.context(a, 0, 1)
    if not a.keyed:
        c.upload_params(*mr.make_params(a.F, a.k, a.model))
    for s in range(steps):
        mr.upload(c, a.model, 0, mr.global_batch([b[s] for b in per_rank]), a.keyed)
        c.train_step(0)
    path = os.path.join(str(tmp_path), name)
    c.save_checkpoint(path)
    snap = wk.snapshot(c, a)
    c.close()
    return path, snap


@pytest.mark.parametrize("keyed", [False, True])
def test_reshard_one_gpu_file_onto_two_ranks(tmp_path, keyed):
    """load_checkpoint_shards([single-GPU file]) on 2 ranks: the global downloads are the single-GPU arrays; keyed, every
    key lives only on its owner, in rows [0, n_r) in source order, and a resident slot is stale until uploaded again"""
    from lightctr_b200 import dist as ldist
    a = _args(keyed=keyed)
    path, single = _single_file(tmp_path, a, "single")
    if keyed:
        np.save(path + ".keys.npy", single["keys"])
    _run(tmp_path, ["--mode", "from1", "--single", path] + _cli(a))
    parts, res = mr.load(tmp_path), mr.load_json(tmp_path)
    F = mr.CAP_MULT * a.F if keyed else a.F
    rowlen = a.k
    for o in res:
        assert np.isfinite(o["after_upload"])
    if not keyed:
        m = _merged(parts, "", F)
        for x in ("W", "V", "s1"):
            assert np.array_equal(_bits(m[x]), _bits(single[x])), x
        return
    keys = single["keys"]
    owner = ldist.owner_of_key(keys, 2)
    for r, (p, o) in enumerate(zip(parts, res)):
        mine = keys[owner == r]
        assert len(mine) > 0 and np.array_equal(p["keys"], mine)
        want = np.full(len(keys), -1, np.int64)
        want[owner == r] = np.arange(len(mine)) * 2 + r
        assert np.array_equal(p["rows"], want)
        assert o["stale"] is not None and "stale" in o["stale"], o["stale"]
        for l, key in enumerate(mine.tolist()):
            i, g = int(np.nonzero(keys == np.uint64(key))[0][0]), l * 2 + r
            assert _bits(np.float32(p["W"][g])) == _bits(np.float32(single["W"][i]))
            assert np.array_equal(_bits(p["V"][g * rowlen:(g + 1) * rowlen]), _bits(single["V"][i * rowlen:(i + 1) * rowlen]))
            assert _bits(np.float32(p["s1"][g])) == _bits(np.float32(single["s1"][i]))


def test_refused_loads_leave_the_context_unchanged(tmp_path):
    from lightctr_b200 import capi, dist as ldist
    a = _args()
    single, _ = _single_file(tmp_path, a, "single", steps=1)
    other, _ = _single_file(tmp_path, _args(k=8), "other_cfg", steps=1)
    # keyed FM, capacity 64: 40 keys all owned by rank 1 under world 2, whose shard holds 32 rows
    c = wk.context(_args(keyed=True, k=8), 0, 1, cap=64)
    pool = ldist.fmix64(np.arange(1, 2000))
    skew = pool[ldist.owner_of_key(pool, 2) == 1][:40]
    c.upload_keyed_params(skew, np.ones(40, np.float32), None)
    skewed = os.path.join(str(tmp_path), "skewed")
    c.save_checkpoint(skewed)
    c.close()
    _run(tmp_path, ["--mode", "refuse", "--single", single, "--other-cfg", other, "--skewed", skewed] + _cli(a))
    res = mr.load_json(tmp_path)
    for r, o in enumerate(res):
        for x in ("other_rank", "single_file", "incomplete", "duplicate", "steps", "cfg", "wnd_layers"):
            assert o[x] != "NOT REFUSED" and not o[x].startswith("CHANGED"), (x, o[x])
        assert "rank %d of world 2" % (1 - r) in o["other_rank"] and "rank %d of world 2" % r in o["other_rank"], o["other_rank"]
        assert "rank 0 of world 1" in o["single_file"], o["single_file"]
        assert "world 2" in o["incomplete"] and "1 files" in o["incomplete"], o["incomplete"]
        assert "appears twice" in o["duplicate"], o["duplicate"]
        assert "step" in o["steps"] and "not one save" in o["steps"], o["steps"]
        assert "different trainer" in o["cfg"], o["cfg"]
        assert "dense layers" in o["wnd_layers"], o["wnd_layers"]
        assert np.isfinite(o["after_load"])
    assert res[0]["keyed_overflow"] == "NOT REFUSED"  # rank 0 receives none of the keys
    msg = res[1]["keyed_overflow"]
    assert "rank 1 would hold 40 keys" in msg and "capacity is 32" in msg and not msg.startswith("CHANGED"), msg
    # a shard file through a single-GPU context's lctr_load_checkpoint
    c = wk.context(a, 0, 1)
    with pytest.raises(capi.LctrError, match="load_checkpoint_shards"):
        c.load_checkpoint(ldist.shard_path(os.path.join(str(tmp_path), "A"), 0, 2))
    c.close()
