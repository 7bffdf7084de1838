"""Frequency admission of keyed contexts (include/lightctr_b200.h: lctr_set_key_admission): the header declares the three
calls, the ctypes binding loads them, and the feature adds nothing to lctr_cfg (reserved[1] stays 0)."""
import ctypes as C
import os
import re

from conftest import ROOT

from lightctr_b200 import build as lbuild
from lightctr_b200 import capi

CALLS = {
    "lctr_set_key_admission": "int lctr_set_key_admission(lctr_ctx* ctx, uint32_t min_count, uint32_t log2_width);",
    "lctr_decay_key_admission": "int lctr_decay_key_admission(lctr_ctx* ctx, uint32_t shift);",
    "lctr_key_admission_stats": "int lctr_key_admission_stats(lctr_ctx* ctx, uint64_t* dropped_entries, uint64_t* admitted_keys);",
}


def test_header_declares_the_admission_calls():
    hdr = open(os.path.join(ROOT, "include", "lightctr_b200.h")).read()
    flat = re.sub(r"\s+", " ", hdr)
    for name, decl in CALLS.items():
        assert decl in flat, name
        assert name in capi.SYMBOLS
    # the sketch's cell formula is stated where a caller can restate it
    assert "fmix64(x ^ ((i + 1) * 0x9E3779B97F4A7C15)) >> (64 - log2_width)" in flat


def test_binding_loads_the_admission_calls():
    lbuild.build()
    L = capi.load_library()
    for name in CALLS:
        assert hasattr(L, name), name
    assert L.lctr_set_key_admission.argtypes == [C.c_void_p, C.c_uint32, C.c_uint32]
    assert L.lctr_decay_key_admission.argtypes == [C.c_void_p, C.c_uint32]
    assert L.lctr_key_admission_stats.argtypes == [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    for m in ("set_key_admission", "decay_key_admission", "key_admission_stats"):
        assert callable(getattr(capi.Context, m))


def test_admission_is_not_part_of_the_cfg():
    cfg = capi.Cfg()
    assert cfg.reserved[1] == 0
    names = [n for n, _ in capi.Cfg._fields_]
    assert not any("admi" in n for n in names)
    hdr = open(os.path.join(ROOT, "include", "lightctr_b200.h")).read()
    assert "uint32_t reserved[2]; /* reserved[1] must stay 0 */" in hdr
