"""cfg.key_evict (include/lightctr_b200.h) took the place of reserved[0]: the struct keeps its size and every other offset,
so there is no ABI version bump, and zero is today's behaviour."""
import ctypes as C
import os
import subprocess
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _offsets(fields):
    src = ('#include "lightctr_b200.h"\n#include <stdio.h>\n#include <stddef.h>\n'
           'int main(){printf("%zu' + ' %zu' * len(fields) + '\\n", sizeof(lctr_cfg)' +
           ''.join(', offsetof(lctr_cfg, %s)' % f for f in fields) + ');return 0;}\n')
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, "s.c")
        open(p, "w").write(src)
        subprocess.check_call(["/usr/bin/gcc", "-I", os.path.join(ROOT, "include"), p, "-o", os.path.join(d, "s")])
        return list(map(int, subprocess.check_output([os.path.join(d, "s")]).split()))


def test_cfg_key_evict_sits_where_reserved0_was():
    from lightctr_b200 import capi
    size, off_ema, off_evict, off_res = _offsets(["ema_rate", "key_evict", "reserved"])

    class OldTail(C.Structure):  # the layout before key_evict: ema_rate then reserved[3]
        _fields_ = [(n, t) for n, t in capi.Cfg._fields_ if n not in ("key_evict", "reserved")] + [("reserved", C.c_uint32 * 3)]

    assert size == C.sizeof(capi.Cfg) == C.sizeof(OldTail)
    assert off_evict == capi.Cfg.key_evict.offset == OldTail.reserved.offset == off_ema + 4
    assert off_res == capi.Cfg.reserved.offset == off_evict + 4
    assert capi.Cfg.reserved.size == 8


def test_cfg_key_evict_defaults_to_off():
    from lightctr_b200 import capi
    assert capi.Cfg().key_evict == 0
    assert "lctr_evict_keys" in capi.SYMBOLS
