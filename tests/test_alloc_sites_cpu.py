"""Every device and pinned allocation of the library goes through one owner, Buf in csrc/common.cuh: no other code in
csrc calls the CUDA allocation or release functions.  The one exception is the process-lifetime trace buffer of
LCTR_MLP_UMMA_TRACE (d_trace in mlp_umma.cu).  cudaIpc* calls map other processes' memory and are not allocations."""
import os
import re

from conftest import ROOT

CSRC = os.path.join(ROOT, "lightctr_b200", "csrc")
ALLOC = re.compile(r"\bcuda(Malloc\w*|HostAlloc|Free|FreeHost)\s*\(")


def _buf_lines(lines):
    """line numbers of the body of `class Buf` in common.cuh"""
    start = next(i for i, l in enumerate(lines) if l.startswith("class Buf {"))
    end = next(i for i in range(start, len(lines)) if lines[i].startswith("};"))
    return range(start, end + 1)


def test_no_allocation_outside_the_buffer_type():
    found = []
    for name in sorted(os.listdir(CSRC)):
        if not name.endswith((".cu", ".cuh", ".cpp", ".h")):
            continue
        lines = open(os.path.join(CSRC, name)).read().splitlines()
        allowed = _buf_lines(lines) if name == "common.cuh" else range(0)
        for i, line in enumerate(lines):
            code = line.split("//")[0]
            if ALLOC.search(code) and i not in allowed and "d_trace" not in code:
                found.append("%s:%d: %s" % (name, i + 1, line.strip()))
    assert not found, "allocation outside Buf:\n" + "\n".join(found)


def test_the_buffer_type_allocates():
    """the check above would pass vacuously if Buf itself moved: it holds the allocation calls"""
    lines = open(os.path.join(CSRC, "common.cuh")).read().splitlines()
    body = "\n".join(lines[i] for i in _buf_lines(lines))
    for call in ("cudaMalloc(", "cudaMallocHost(", "cudaHostAlloc(", "cudaFree(", "cudaFreeHost("):
        assert call in body, call
