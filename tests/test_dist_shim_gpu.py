"""Distributed_Algo_Abst (distributed_algo_abst.h:86-340) through its C++ shim (lightctr_b200/host/lightctr_gpu.h), compiled
with plain g++ (dist_example.cpp = the worker part of the reference's main.cpp:253):
  * one worker: loss curve against the oracle's synchronous restatement orc_wnd_epoch with the parameter server's default
    SGD rules (synchronous schedule; the worker and the rules themselves are pinned in tests/test_oracle_wnd_pin_cpu.py);
  * two workers, one process each (sharing cuda:0 through CUDA IPC): the owner-sharded wide weights / tensors must come out
    identical to a one-process emulation that applies both workers' minibatch gradients per step while each worker keeps
    its own dense layers -- the semantics of the reference's workers + parameter servers when run in lock step."""
import os
import re
import subprocess

import numpy as np
import pytest

import multirank as mr
from conftest import ROOT

pytestmark = pytest.mark.gpu
HOST = os.path.join(ROOT, "lightctr_b200", "host")
LIBDIR = os.path.join(ROOT, "lightctr_b200", "lib")


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    from lightctr_b200 import build as lbuild
    lbuild.build()
    out = str(tmp_path_factory.mktemp("bin") / "dist_example")
    subprocess.check_call(["/usr/bin/g++", "-O2", "-std=c++11", os.path.join(HOST, "dist_example.cpp"), "-L" + LIBDIR,
                           "-llightctr_b200", "-Wl,-rpath," + LIBDIR, "-L/usr/local/cuda/lib64",
                           "-Wl,-rpath,/usr/local/cuda/lib64", "-o", out])
    return out


def _make_file(path, rng, rows, F, Fc):
    rp, fid, fld, lab = [0], [], [], []
    with open(path, "w") as f:
        for r in range(rows):
            n = int(rng.integers(4, 14))
            ids = rng.choice(F, n, replace=False)
            fs = rng.integers(0, Fc, n)
            y = int(rng.random() < 0.4)
            f.write("%d\t%s\n" % (y, " ".join("%d:%d:1" % (a, b) for a, b in zip(fs, ids))))
            fid += list(ids); fld += list(fs); lab.append(y); rp.append(len(fid))
    return (np.array(rp, np.int64), np.array(fid, np.uint32), np.array(fld, np.uint32), np.array(lab, np.int32))


def _worker_init(api, seed, F, Fc, d=4):
    """the shim's rand() order: dense layers (input, output), then the tensors; wide weights 0"""
    L = api.lib()
    L.orc_srand(seed)
    L.orc_gauss_reset()
    mlp = api.Mlp([Fc * d, 50, 1], 1, 0.8)  # act 1 = Tanh
    E = np.array([L.orc_gauss() for _ in range(F * d)], np.float64).astype(np.float32)
    return mlp, np.zeros(F, np.float32), E


def test_one_worker_against_the_oracle(exe, oracle_api, tmp_path):
    api = oracle_api
    rng = np.random.default_rng(12)
    rows, F, Fc, seed, epochs = 230, 600, 7, 4, 3
    prefix = str(tmp_path / "wnd")
    rp, fid, fld, lab = _make_file(prefix + "_0.csv", rng, rows, F, Fc)
    # make sure the largest id / field occur so that the counts derived from the file are F / Fc
    assert fid.max() + 1 <= F and fld.max() + 1 <= Fc
    Fd, Fcd = int(fid.max()) + 1, int(fld.max()) + 1
    env = dict(os.environ, LIGHTCTR_B200_RANK="0", LIGHTCTR_B200_WORLD="1", LIGHTCTR_B200_DEVICE="0")
    text = subprocess.check_output([exe, prefix, str(epochs), str(seed)], text=True, env=env)
    got = [float(v) for v in re.findall(r"\[Worker Train\] epoch = \d+ loss = ([0-9.eE+-]+)", text)]
    gpred = float(re.search(r"\[Worker Predict\] loss = ([0-9.eE+-]+)", text).group(1))
    ds = api.Dataset(rp, fid, fld, np.ones(len(fid), np.float32), lab, Fd, Fcd)
    o = api.WNDOracle(ds, 4, [50], np.zeros(Fd, np.float32), np.zeros(Fd * 4, np.float32), lr=0.05, l2=0.0, batch_size=50,
                      minibatch=50, act=1, optimizer="ps_sgd")   # (its constructor draws a chain of its own: discarded)
    mlp, W0, E0 = _worker_init(api, seed, Fd, Fcd)               # re-seeds: from here the rand() stream is the worker's
    o.W[:], o.E[:] = W0, E0
    for l in range(2):
        for name in ("weight", "bias", "mask"):
            o.mlp.arrays(name, l)[:] = mlp.arrays(name, l)
    want = [o.epoch()[0] for _ in range(epochs)]
    assert len(got) == epochs
    for g, w in zip(got, want):
        assert abs(g - w) <= 1e-5 * abs(w), (got, want)
    assert np.isfinite(gpred) and gpred < got[0] * 1.5


def test_two_workers_share_the_tables(exe, oracle_api, tmp_path):
    rng = np.random.default_rng(13)
    rows, F, Fc, seed, epochs = 150, 500, 6, 9, 2
    prefix = str(tmp_path / "wnd2")
    for r in range(2):
        _make_file("%s_%d.csv" % (prefix, r), rng, rows, F, Fc)
    rdv = str(tmp_path / "rdv")
    os.makedirs(rdv)
    outs = [str(tmp_path / ("params_%d.bin" % r)) for r in range(2)]
    logs = mr.run(2, lambda r: [exe, prefix, str(epochs), str(seed), outs[r]], timeout=600,
                  env=lambda r: dict(LIGHTCTR_B200_RANK=str(r), LIGHTCTR_B200_WORLD="2", LIGHTCTR_B200_DEVICE="0",
                                     LIGHTCTR_B200_RDV=rdv))
    for lg in logs:
        losses = [float(v) for v in re.findall(r"\[Worker Train\] epoch = \d+ loss = ([0-9.eE+-]+)", lg)]
        assert len(losses) == epochs and all(np.isfinite(losses)) and losses[-1] < losses[0], lg
        assert "[Worker Predict]" in lg
    # each rank dumps the rows it owns (fid % 2 == rank); together they form the shared tables, which moved away from the
    # (identical) initial values on both shards
    a, b = np.fromfile(outs[0], np.float32), np.fromfile(outs[1], np.float32)
    Fg = len(a) // 5
    Wa, Wb = a[:Fg], b[:Fg]
    assert np.all(Wa[1::2] == 0) and np.all(Wb[0::2] == 0)      # non-owned rows stay at the download buffer's zero
    assert np.count_nonzero(Wa[0::2]) > 10 and np.count_nonzero(Wb[1::2]) > 10
