"""The collective score (csrc/capi.cu: lctr_score on world > 1): 2 ranks sharing cuda:0 over CUDA IPC
(tests/dist_score_worker.py), against the ranks' own train steps and a single-GPU context of the same cfg holding the
merged parameters."""
import argparse

import numpy as np
import pytest

import dist_score_worker as wk
import multirank as mr

pytestmark = pytest.mark.gpu
TOL = 1e-5  # parameters and losses of two sharded runs: the sparse scatter sums in arbitrary order


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def _reference_score(args, parts, rank, test):
    """world-1 context of the same cfg holding the merged W / V and the rank's dense layers: the score of its test batch"""
    from lightctr_b200 import dist as ldist
    ctx = wk.context(args, 0, 1)
    ctx.upload_params(ldist.merge_shards([p["W"] for p in parts], 2, args.F),
                      ldist.merge_shards([p["V"] for p in parts], 2, args.F))
    for l in range(len(wk.layer_dims(args)) - 1):
        ctx.mlp_upload(l, parts[rank]["mlp_w%d" % l], parts[rank]["mlp_b%d" % l])
    mr.upload(ctx, args.model, 1, test)
    out = ctx.score(1)
    ctx.close()
    return out


@pytest.mark.parametrize("model,k,flags", [("fm", 16, ["--empty"]), ("ffm", 4, []), ("nfm", 16, ["--empty"]),
                                           ("nfm", 16, ["--bf16"]), ("wnd", 4, ["--empty"]), ("fm", 16, ["--keyed"]),
                                           ("nfm", 16, ["--keyed", "--bf16", "--empty"])],
                         ids=["fm-empty", "ffm", "nfm_fp32-empty", "nfm_bf16", "wnd-empty", "fm-keyed", "nfm_bf16-keyed-empty"])
def test_collective_score(tmp_path, model, k, flags):
    """each rank's score of a train batch equals the pred of the train step that follows it, bit for bit; the score of its
    test batch (empty on rank 1 with --empty) equals a world-1 context holding the merged parameters (Wide&Deep: the rank's
    own dense layers, to 1e-6 as lctr_predict's); dist.eval_global after the score equals lctr_eval_pred on the
    concatenation; and the steps after a score follow the run without scores"""
    from lightctr_b200 import capi
    argv = ["--model", model, "--k", str(k)] + flags
    out = str(tmp_path)
    mr.launch("dist_score_worker.py", out, argv)
    parts, res = mr.load(out), mr.load_json(out)
    args = argparse.Namespace(model=model, k=k, F=20000, rows=256, test_rows=200, bf16="--bf16" in flags,
                              keyed="--keyed" in flags, empty="--empty" in flags)
    tests = [mr.test_batches(args.F, args.test_rows, 1, r)[0] if not (args.empty and r == 1) else wk.empty_batch()
             for r in range(2)]
    for r in range(2):
        p = parts[r]
        for i in range(3):
            assert _bits(p["s%d" % i]).tolist() == _bits(p["p%d" % i]).tolist(), (r, i)
        assert len(p["test"]) == len(tests[r][3])
        if not args.keyed:
            ref = _reference_score(args, parts, r, tests[r])
            if model == "wnd":
                assert np.allclose(p["test"], ref, rtol=1e-6, atol=0), r
            else:
                assert _bits(p["test"]).tolist() == _bits(ref).tolist(), (r, np.max(np.abs(p["test"] - ref), initial=0))
        assert np.allclose(res[r]["loss"], res[r]["n_loss"], rtol=TOL, atol=0), (r, res[r]["loss"], res[r]["n_loss"])
    probe = capi.Context(capi.MODEL_FM, 10, 4)
    want = probe.eval_pred(np.concatenate([parts[r]["test"] for r in range(2)]),
                           np.concatenate([parts[r]["test_label"] for r in range(2)]))
    probe.close()
    for r in range(2):
        assert res[r]["eval"] == list(want), (r, res[r]["eval"], want)
    if not args.keyed:
        from lightctr_b200 import dist as ldist
        for a, b in (("W_end", "n_W_end"), ("V_end", "n_V_end")):
            x = ldist.merge_shards([p[a] for p in parts], 2, args.F)
            y = ldist.merge_shards([p[b] for p in parts], 2, args.F)
            assert np.max(np.abs(x - y)) < TOL, a
