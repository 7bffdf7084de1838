"""Build the sm_90a shared library (lightctr_b200/lib/liblightctr_b200.so) with nvcc, in-tree.

    python -m lightctr_b200.build [--force] [--verbose]
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib", "liblightctr_b200.so")
SOURCES = ["capi.cu", "fm.cu", "fm_fused.cu", "ffm.cu", "ffm_warp.cu", "ffm_grouped.cu", "opt.cu", "mlp.cu", "mlp_bf16.cu", "mlp_umma.cu", "dist.cu", "csc.cu", "checkpoint.cu", "metrics.cu", "wnd.cu", "keys.cu", "text.cu", "loader.cpp"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
# -fmad=false: the reference is built without FMA (-mavx only, Makefile:3); keeping mul and add
# separately rounded keeps per-coordinate updates comparable bit-for-bit.  All kernels here are
# memory-bound, so contraction would buy nothing.
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-fmad=false",
         "-ccbin", "/usr/bin/g++", "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function", "-shared", "-cudart", "shared"]


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "lightctr_b200.h"),
                                                               os.path.abspath(__file__)]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    os.makedirs(os.path.dirname(LIB), exist_ok=True)
    cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if verbose or r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed building %s" % LIB)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
