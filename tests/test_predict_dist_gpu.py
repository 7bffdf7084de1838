"""Collective predict and global test metrics on multi-GPU trainers (csrc/capi.cu: predict_dist, csrc/dist.cu: pull-only
rounds and the cache release, lightctr_b200/dist.py: eval_global): 2 ranks sharing cuda:0 over CUDA IPC against a
single-GPU context of the same cfg holding the merged parameters."""
import numpy as np
import pytest

import dist_predict_worker as wk
import multirank as mr

pytestmark = pytest.mark.gpu
TOL = 1e-5  # parameters of two sharded runs: the sparse scatter sums in arbitrary order


def _run(out, extra):
    mr.launch("dist_predict_worker.py", out, extra)
    return mr.load(out), mr.load_json(out)


def _merged(parts, F, wkey="W", vkey="V"):
    from lightctr_b200 import dist as ldist
    return (ldist.merge_shards([p[wkey] for p in parts], 2, F), ldist.merge_shards([p[vkey] for p in parts], 2, F))


def _reference_pctr(model, F, k, rows, W, V, batches):
    """world-1 context of the same cfg holding W / V: the pCTR of each batch"""
    ctx = wk.context(model, F, k, 0, 1, rows)
    ctx.upload_params(W, V)
    out = []
    for b in batches:
        mr.upload(ctx, model, 1, b)
        out.append(ctx.predict(1))
    ctx.close()
    return out


def _same_bits(a, b):
    return a.shape == b.shape and np.array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("model,k", [("fm", 16), ("ffm", 4)])
def test_predict_parity_with_merged_single_gpu(tmp_path, model, k):
    """FM k=16 Adagrad / FFM k=4 on 39 fields, 3 train steps on 2 ranks, then each rank predicts its own test batch: bit for
    bit the pCTR of a world-1 context holding the merged parameters"""
    F, rows, test_rows = 20000, 256, 200
    parts, _ = _run(str(tmp_path), ["--mode", "parity", "--model", model, "--k", str(k), "--F", str(F), "--rows", str(rows),
                                    "--test-rows", str(test_rows)])
    W, V = _merged(parts, F)
    tests = [mr.test_batches(F, test_rows, 1, r)[0] for r in range(2)]
    ref = _reference_pctr(model, F, k, rows, W, V, tests)
    for r in range(2):
        assert len(parts[r]["pctr"]) == test_rows
        assert _same_bits(parts[r]["pctr"], ref[r]), (r, np.max(np.abs(parts[r]["pctr"] - ref[r])))


def test_predict_interleaved_with_training(tmp_path):
    """train, predict twice, train, predict two slots, train: repeated predicts agree bit for bit, each equals the world-1
    pCTR at the parameters of that moment, and the predicts leave training unchanged; a step after a predict launches one
    kernel more than the same step after a train step (the wait for the released caches)"""
    F, k, rows, test_rows = 20000, 16, 256, 200
    with_p, _ = _run(str(tmp_path / "p"), ["--mode", "interleave", "--model", "fm", "--k", str(k), "--rows", str(rows),
                                           "--test-rows", str(test_rows)])
    without, _ = _run(str(tmp_path / "n"), ["--mode", "interleave", "--model", "fm", "--k", str(k), "--rows", str(rows),
                                            "--test-rows", str(test_rows), "--no-predict"])
    tests = [mr.test_batches(F, test_rows, 2, r) for r in range(2)]
    W0, V0 = _merged(with_p, F, "W0", "V0")
    W1, V1 = _merged(with_p, F, "W1", "V1")
    ref0 = _reference_pctr("fm", F, k, rows, W0, V0, [tests[r][0] for r in range(2)])
    ref1 = _reference_pctr("fm", F, k, rows, W1, V1, [t for r in range(2) for t in tests[r]])
    for r in range(2):
        p = with_p[r]
        assert _same_bits(p["p1a"], p["p1b"])
        assert _same_bits(p["p1a"], ref0[r])
        assert _same_bits(p["p2_1"], ref1[2 * r]) and _same_bits(p["p2_2"], ref1[2 * r + 1])
    for i in range(3):
        a, b = _merged(with_p, F, "W%d" % i, "V%d" % i), _merged(without, F, "W%d" % i, "V%d" % i)
        assert np.max(np.abs(a[0] - b[0])) < TOL and np.max(np.abs(a[1] - b[1])) < TOL, i
    for r in range(2):
        lp, ln = with_p[r]["launches"], without[r]["launches"]
        assert lp[0] == ln[0] and lp[1] == ln[1] + 1 and lp[2] == ln[2] + 1, (lp, ln)
        assert list(lp) == [7, 8, 8] and list(ln) == [7, 7, 7], (r, list(lp), list(ln))


def test_wnd_predict_twice_then_train(tmp_path):
    """Wide&Deep: two predicts in a row give the same bits; a train step and a third predict run to the end"""
    parts, res = _run(str(tmp_path), ["--mode", "wnd", "--k", "4", "--rows", "128", "--test-rows", "100"])
    for p, o in zip(parts, res):
        assert len(p["p1a"]) == 100 and _same_bits(p["p1a"], p["p1b"])
        assert np.isfinite(o["loss"]) and np.all(np.isfinite(p["p2"]))


@pytest.mark.parametrize("model,k", [("fm", 16), ("ffm", 4), ("wnd", 4), ("nfm", 16)])
def test_empty_share_predicts_and_trains(tmp_path, model, k):
    """rank 1 uploads 0 rows: both ranks predict (rank 1 gets an empty array; NFM has no predictor), and a train step with
    rank 1 contributing no gradients equals a world-1 step on rank 0's rows -- dense layers included: NFM's all-reduce
    still runs on the empty rank (both ranks end with the world-1 layers), Wide&Deep's per-rank layers stay as they were
    on the empty rank"""
    F, rows, test_rows = 20000, 256, 200
    parts, res = _run(str(tmp_path), ["--mode", "empty", "--model", model, "--k", str(k), "--rows", str(rows),
                                      "--test-rows", str(test_rows)])
    assert res[1]["stats"] == [0.0, 0.0]
    W0, V0 = mr.make_params(F, k, model)
    dense = mr.dense_layers(model, k)
    if model != "nfm":
        assert len(parts[1]["pctr"]) == 0 and len(parts[1]["pctr_after"]) == 0
        test0 = mr.test_batches(F, test_rows, 1, 0)[0]
        ctx = wk.context(model, F, k, 0, 1, rows)
        ctx.upload_params(W0, V0)
        for l, (w, b) in enumerate(dense):
            ctx.mlp_upload(l, w, b)
        mr.upload(ctx, model, 1, test0)
        ref = ctx.predict(1)
        ctx.close()
        if model == "wnd":
            assert np.allclose(parts[0]["pctr"], ref, rtol=1e-6, atol=0)
        else:
            assert _same_bits(parts[0]["pctr"], ref)
    ctx = wk.context(model, F, k, 0, 1, rows)
    ctx.upload_params(W0, V0)
    for l, (w, b) in enumerate(dense):
        ctx.mlp_upload(l, w, b)
    mr.upload(ctx, model, 0, mr.train_batches(F, rows, 1, 0)[0])
    loss, correct = ctx.train_step(0)
    W, V = ctx.download_params()
    dims = mr.layer_dims(model, k)
    layers = [ctx.mlp_download(l, dims[l], dims[l + 1]) for l in range(len(dims) - 1)]
    ctx.close()
    got_loss, got_correct = res[0]["reduced"]
    assert abs(got_loss - loss) <= 1e-5 * abs(loss) and got_correct == correct
    Wg, Vg = _merged(parts, F)
    assert np.max(np.abs(Wg - W)) < TOL and np.max(np.abs(Vg - V)) < TOL
    for l, (w, b) in enumerate(layers):
        assert np.max(np.abs(parts[0]["mlp_w%d" % l] - w)) < TOL and np.max(np.abs(parts[0]["mlp_b%d" % l] - b)) < TOL, l
        if model == "nfm":  # replicated layers: the all-reduce gave rank 1 rank 0's gradients
            assert np.array_equal(parts[1]["mlp_w%d" % l], parts[0]["mlp_w%d" % l])
            assert np.array_equal(parts[1]["mlp_b%d" % l], parts[0]["mlp_b%d" % l])
        else:  # per-rank layers: no row, no gradient, no update
            w0, b0 = dense[l]
            assert np.array_equal(parts[1]["mlp_w%d" % l], w0.reshape(-1)) and np.array_equal(parts[1]["mlp_b%d" % l], b0)


def test_keyed_predict_parity_with_merged_single_gpu(tmp_path):
    """keyed FM k=16 (slots uploaded with insert = 1): 3 train steps on 2 ranks, then each rank predicts its own test batch;
    bit for bit the pCTR of a world-1 keyed context seeded with the merged key -> (W, V) map (dist.merge_keyed_shards)"""
    from lightctr_b200 import dist as ldist
    F, k, rows, test_rows = 20000, 16, 256, 200
    parts, _ = _run(str(tmp_path), ["--mode", "parity", "--model", "fm", "--k", str(k), "--F", str(F), "--rows", str(rows),
                                    "--test-rows", str(test_rows), "--keyed"])
    got = ldist.merge_keyed_shards([p["keys"] for p in parts], [p["W"] for p in parts], [p["V"] for p in parts], 2)
    keys = np.array(sorted(got), np.uint64)
    ctx = wk.context("fm", F, k, 0, 1, rows, keyed=True)
    ctx.upload_keyed_params(keys, np.array([got[int(x)][0] for x in keys], np.float32),
                            np.concatenate([got[int(x)][1] for x in keys]).astype(np.float32))
    for r in range(2):
        rp, fid, _, lab = mr.test_batches(F, test_rows, 1, r)[0]
        ctx.upload_batch_keys(1, rp, ldist.fmix64(fid), None, None, lab, insert=False)  # every key is in the merged map
        ref = ctx.predict(1)
        assert len(parts[r]["pctr"]) == test_rows
        assert _same_bits(parts[r]["pctr"], ref), (r, np.max(np.abs(parts[r]["pctr"] - ref)))
    ctx.close()


def test_empty_share_keyed_upload(tmp_path):
    """a keyed collective upload with one empty share posts empty lists: the upload, a train step and the predicts complete"""
    parts, res = _run(str(tmp_path), ["--mode", "empty", "--model", "fm", "--k", "16", "--keyed"])
    assert len(parts[1]["pctr"]) == 0 and res[1]["stats"] == [0.0, 0.0]
    for key in ("pctr", "pctr_after"):
        p = parts[0][key]
        assert len(p) == 200 and np.all((p > 0) & (p < 1))
    assert np.isfinite(res[0]["stats"][0]) and res[0]["reduced"] == res[0]["stats"]
    assert len(parts[0]["keys"]) + len(parts[1]["keys"]) > 0


@pytest.mark.parametrize("shares", ["300,170", "0,300"])
def test_eval_global_equals_single_gpu_eval(tmp_path, shares):
    """dist.eval_global over uneven shares (one of them empty): the same numbers on every rank, bit for bit lctr_eval of a
    world-1 context holding the concatenated batch with the same pCTR -- predicted, and crafted with ties and values
    sharing a bucket"""
    F, k, rows = 20000, 16, 256
    n = [int(x) for x in shares.split(",")]
    parts, res = _run(str(tmp_path), ["--mode", "metrics", "--model", "fm", "--k", str(k), "--rows", str(rows),
                                      "--test-rows-per-rank", shares])
    assert res[0]["predicted"] == res[1]["predicted"] and res[0]["crafted"] == res[1]["crafted"]
    for o in res:  # rank 1's label count did not match: both ranks raised
        assert o["mismatch"] is not None and "rank(s) [1]" in o["mismatch"], o["mismatch"]
    ctx = wk.context("fm", F, k, 0, 1, rows)
    mr.upload(ctx, "fm", 1, mr.global_batch([mr.test_batches(F, n[r], 1, r)[0] for r in range(2) if n[r]]))
    for key in ("pctr", "crafted"):
        ctx.upload_pred(1, np.concatenate([parts[r][key] for r in range(2)]))
        want = ctx.eval_metrics(1)
        got = res[0]["predicted" if key == "pctr" else "crafted"]
        assert np.float32(got[0]).view(np.uint32) == np.float32(want[0]).view(np.uint32), (key, got, want)
        assert got[1] == want[1], (key, got, want)
        assert np.float32(got[2]).view(np.uint32) == np.float32(want[2]).view(np.uint32), (key, got, want)
    ctx.close()


def test_eval_pred_equals_eval_single_gpu():
    """lctr_eval_pred over host arrays equals lctr_eval on the slot holding the same pCTR and labels, bit for bit"""
    F, k, rows = 20000, 16, 3000
    b = mr.test_batches(F, rows, 1, 0)[0]
    ctx = wk.context("fm", F, k, 0, 1, rows)
    ctx.upload_params(*mr.make_params(F, k, "fm"))
    mr.upload(ctx, "fm", 1, b)
    pred = ctx.predict(1)
    for p in (pred, wk.crafted_pctr(rows, 0)):
        ctx.upload_pred(1, p)
        want = ctx.eval_metrics(1)
        got = ctx.eval_pred(p, b[3])
        assert np.float32(got[0]).view(np.uint32) == np.float32(want[0]).view(np.uint32)
        assert got[1] == want[1]
        assert np.float32(got[2]).view(np.uint32) == np.float32(want[2]).view(np.uint32)
    with pytest.raises(Exception, match="no rows"):
        ctx.eval_pred(np.zeros(0, np.float32), np.zeros(0, np.int32))
    ctx.close()


def test_predict_refusals_on_two_ranks(tmp_path):
    """the quirk predictor is refused on world > 1 with its reason (and the context predicts afterwards), NFM keeps its
    message, and a test batch whose per-owner key list outgrew its inbox fails with the overflow message"""
    parts, res = _run(str(tmp_path), ["--mode", "refuse", "--k", "16", "--rows", "128", "--test-rows", "100"])
    for p, o in zip(parts, res):
        assert o["quirk"] is not None and "quirk_sumvx_slot is single-GPU" in o["quirk"], o["quirk"]
        assert len(p["after_quirk"]) == 100 and np.all(np.isfinite(p["after_quirk"]))
        assert o["nfm"] is not None and "ships no NFM predictor" in o["nfm"], o["nfm"]
    assert res[0]["overflow"] is not None and "outgrew its inbox" in res[0]["overflow"], res[0]["overflow"]
    assert res[1]["overflow"] is None
