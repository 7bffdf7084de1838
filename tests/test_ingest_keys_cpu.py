"""Host-side keyed ingest: lctr_load_libffm_keys is the dense loader's parser with ids kept at their full 64-bit width.
On the committed fixtures it gives the dense loader's CSR (with key == fid) including the reference parser's quirks;
ids >= 2^32 parse exactly where the dense loader rejects them.  No GPU needed: these entry points are host code."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from golden_util import GOLDEN, load_csr, write_libffm


@pytest.fixture(scope="module")
def capi():
    from lightctr_b200 import build as lbuild
    from lightctr_b200 import capi as _capi
    lbuild.build()
    _capi.load_library()
    return _capi


def _same_as_dense(capi, path, fc):
    a = capi.load_libffm(path, field_cnt=fc)
    b = capi.load_libffm_keys(path, field_cnt=fc)
    assert (a.rows, a.nnz, a.field_cnt) == (b.rows, b.nnz, b.field_cnt)
    assert np.array_equal(a.row_ptr, b.row_ptr)
    assert np.array_equal(a.fid.astype(np.uint64), b.key)
    assert np.array_equal(a.field, b.field)
    assert np.array_equal(a.val.view(np.uint32), b.val.view(np.uint32))
    assert np.array_equal(a.label, b.label)  # label_cnt >= rows: the label shift of empty rows is kept
    return b


def test_keyed_loader_matches_dense_on_train_fixture(capi, tmp_path):
    ds = load_csr("train_sparse_csr.npz", field_cnt=68)
    p = str(tmp_path / "train.txt")
    write_libffm(ds, p)
    b = _same_as_dense(capi, p, 68)
    assert (b.rows, b.nnz) == (1000, 281975)


def test_keyed_loader_matches_dense_on_test_head(capi):
    _same_as_dense(capi, os.path.join(GOLDEN, "test_sparse_head.csv"), 0)


def test_keyed_loader_keeps_parser_quirks(capi, tmp_path):
    """empty rows shift the labels, a two-field token keeps the previous value (fm_algo_abst.h:90-103)"""
    p = str(tmp_path / "q.txt")
    open(p, "w").write("1\t0:3:1 1:7:0.5\n1\t\n0\t5:9:1.25 6:10 7:12:3\n-1\t0:0:1e-3 1:1:-2.5\n")
    b = _same_as_dense(capi, p, 3)
    assert len(b.label) == 4 and b.rows == 3
    assert b.val[3] == np.float32(1.25)  # "6:10" reuses the value of the token before it


def test_wide_ids_parse_exactly(capi, tmp_path):
    big = [2 ** 32, 2 ** 32 + 12345, 2 ** 63 + 7, 2 ** 64 - 2, 18446744073709551614, 123]
    p = str(tmp_path / "wide.txt")
    with open(p, "w") as f:
        f.write("1\t0:%d:1 1:%d:0.5 2:%d:2\n" % tuple(big[:3]))
        f.write("0\t3:%d:1 4:%d:1 5:%d:1" % tuple(big[3:]))
    b = capi.load_libffm_keys(p, field_cnt=6)
    assert b.key.tolist() == big
    assert b.row_ptr.tolist() == [0, 3, 6] and b.field.tolist() == [0, 1, 2, 3, 4, 5]
    assert b.val.tolist() == [1.0, 0.5, 2.0, 1.0, 1.0, 1.0] and b.label.tolist() == [1, 0]
    with pytest.raises(capi.LctrError, match="exceed the device index types"):
        capi.load_libffm(p, field_cnt=6)


def test_keyed_dataset_struct_layout_matches_header(capi):
    src = ('#include "lightctr_b200.h"\n#include <stdio.h>\n#include <stddef.h>\n'
           'int main(){printf("%zu %zu %zu\\n", sizeof(lctr_keyed_dataset), offsetof(lctr_keyed_dataset, key), '
           'offsetof(lctr_keyed_dataset, label));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.c")
        open(p, "w").write(src)
        subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), p, "-o", os.path.join(d, "s")])
        size, off_key, off_label = map(int, subprocess.check_output([os.path.join(d, "s")]).split())
    K = capi.KeyedDatasetC
    assert size == C.sizeof(K) and off_key == K.key.offset and off_label == K.label.offset


def test_cfg_key_mode_sits_in_the_old_reserved_slot(capi):
    """key_mode took the place of reserved0: same size and offsets, zero = the dense behaviour (no ABI version bump)"""
    src = ('#include "lightctr_b200.h"\n#include <stdio.h>\n#include <stddef.h>\n'
           'int main(){printf("%zu %zu %zu\\n", sizeof(lctr_cfg), offsetof(lctr_cfg, key_mode), offsetof(lctr_cfg, csc_row_block));return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.c")
        open(p, "w").write(src)
        subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), p, "-o", os.path.join(d, "s")])
        size, off, off_next = map(int, subprocess.check_output([os.path.join(d, "s")]).split())
    assert size == C.sizeof(capi.Cfg) and off == capi.Cfg.key_mode.offset and off_next == off + 4
    assert capi.Cfg().key_mode == capi.KEYS_DENSE == 0
