"""Checkpoints of sharded trainers, host side: the file names of a save (dist.shard_path), the discovery load_sharded runs
on them, and the header reader save_sharded checks the steps with."""
import os
import struct

import pytest

from lightctr_b200 import dist as ldist


def _touch(path, data=b""):
    with open(path, "wb") as f:
        f.write(data)


def test_shard_path_names_rank_and_world(tmp_path):
    p = str(tmp_path / "ckpt")
    assert ldist.shard_path(p, 1, 4) == p + ".rank1-of-4"
    assert ldist.shard_path(p, 0, 1) == p + ".rank0-of-1"


def test_find_shards_rank_order_and_source_world(tmp_path):
    p = str(tmp_path / "ckpt")
    for r in (3, 0, 2, 1):
        _touch(ldist.shard_path(p, r, 4))
    _touch(p + ".rank1-of-4.tmp")           # an interrupted write is not part of the save
    _touch(str(tmp_path / "ckpt2.rank0-of-1"))  # nor is a save under another prefix
    paths, world = ldist.find_shards(p)
    assert world == 4
    assert paths == [ldist.shard_path(p, r, 4) for r in range(4)]
    q = str(tmp_path / "ckpt2")
    assert ldist.find_shards(q) == ([q + ".rank0-of-1"], 1)


def test_find_shards_refuses_gaps_duplicates_and_mixed_worlds(tmp_path):
    p = str(tmp_path / "gap")
    _touch(ldist.shard_path(p, 0, 4))
    _touch(ldist.shard_path(p, 2, 4))
    _touch(ldist.shard_path(p, 3, 4))
    with pytest.raises(ValueError, match=r"ranks \[1\] missing"):
        ldist.find_shards(p)
    d = str(tmp_path / "dup")
    _touch(d + ".rank0-of-2")
    _touch(d + ".rank1-of-2")
    _touch(d + ".rank01-of-2")
    with pytest.raises(ValueError, match="appears twice"):
        ldist.find_shards(d)
    m = str(tmp_path / "mixed")
    _touch(ldist.shard_path(m, 0, 2))
    _touch(ldist.shard_path(m, 1, 2))
    _touch(ldist.shard_path(m, 0, 1))
    with pytest.raises(ValueError, match="several saves"):
        ldist.find_shards(m)
    with pytest.raises(FileNotFoundError):
        ldist.find_shards(str(tmp_path / "none"))


def _header(magic, step, adam_iter, shard=None):
    h = magic + struct.pack("<4i", 1, 0, 0, 0) + struct.pack("<5Q", 100, 0, 16, adam_iter, step) + b"\0" * 72
    assert len(h) == 136
    if shard is not None:
        h += struct.pack("<iiQQ", shard[0], shard[1], 100, 50)
    return h


def test_checkpoint_info_reads_both_formats(tmp_path):
    one = str(tmp_path / "one")
    _touch(one, _header(b"LCTRCKP1", 7, 3))
    assert ldist.checkpoint_info(one) == (7, 3, 1, 0)
    sh = str(tmp_path / "sh")
    _touch(sh, _header(b"LCTRCKS1", 9, 2, shard=(2, 1)))
    assert ldist.checkpoint_info(sh) == (9, 2, 2, 1)
    bad = str(tmp_path / "bad")
    _touch(bad, b"NOTACKPT" + b"\0" * 200)
    with pytest.raises(ValueError, match="not a lightctr_b200 checkpoint"):
        ldist.checkpoint_info(bad)


def test_header_declares_the_shard_loader():
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = open(os.path.join(root, "include", "lightctr_b200.h")).read()
    assert "int lctr_load_checkpoint_shards(lctr_ctx* ctx, int n, const char* const* paths);" in hdr
