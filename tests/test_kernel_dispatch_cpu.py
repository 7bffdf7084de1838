"""Every launcher turns its run-time values into a kernel template instance through by_flags / by_value of
csrc/launch.cuh, which hand a generic lambda compile-time constants that name the instance.  No statement picks among more
than two instances of a __global__ template with ?: chains, and no switch or macro returns one instance per case: a
slip in such a tower compiles and runs an existing instance that is wrong for the combination (unweighted, forward-only,
the wrong HV), which only a bit-exact test of that exact combination would catch.  A single two-way ?: stays."""
import os
import re

from conftest import ROOT

CSRC = os.path.join(ROOT, "lightctr_b200", "csrc")
# template <...> __global__ void [__launch_bounds__(...)] name(
GLOBAL_TEMPLATE = re.compile(r"template\s*<[^;{]*?>\s*__global__\s+void\s+(?:__launch_bounds__\((?:[^()]|\([^()]*\))*\)\s*)?"
                             r"(\w+)\s*\(")
# `case X: return f<...>` / `default: rc = f<...>`: one template instance per case, in a switch or in a macro's cases
CASE_INSTANCE = re.compile(r"\b(?:case\s+[^:;]+|default)\s*:\s*(?:return\s+|\w+\s*=\s*)[\w:]+\s*<")
DEFINE_INSTANCE = re.compile(r"(?:return\s+|=\s*)[\w:]+\s*<")


def _sources(csrc=CSRC):
    for name in sorted(os.listdir(csrc)):
        if name.endswith((".cu", ".cuh")):
            text = open(os.path.join(csrc, name)).read()
            text = re.sub(r"/\*.*?\*/", lambda m: re.sub(r"[^\n]", " ", m.group(0)), text, flags=re.S)
            yield name, re.sub(r"//[^\n]*", "", text)


def _global_templates(csrc=CSRC):
    return {k for _, text in _sources(csrc) for k in GLOBAL_TEMPLATE.findall(text)}


def ternary_towers(csrc=CSRC):
    """statements that name more than two instances of one __global__ template and choose among them with ?:"""
    kernels = _global_templates(csrc)
    found = []
    for name, text in _sources(csrc):
        pos = 0
        for stmt in text.split(";"):
            line = text.count("\n", 0, pos) + 1
            pos += len(stmt) + 1
            if "?" not in stmt:
                continue
            for k in kernels:
                n = len(re.findall(r"\b%s\s*<" % k, stmt))
                if n > 2:
                    found.append("%s:%d: %d instances of %s" % (name, line + stmt.count("\n", 0, len(stmt) - len(stmt.lstrip())), n, k))
    return found


def case_dispatch(csrc=CSRC):
    """switch cases and macros outside launch.cuh that return one template instance per case"""
    found = []
    for name, text in _sources(csrc):
        if name == "launch.cuh":
            continue
        lines = text.replace("\\\n", " ").splitlines()
        for i, line in enumerate(lines):
            if CASE_INSTANCE.search(line) or (line.lstrip().startswith("#define") and DEFINE_INSTANCE.search(line)):
                found.append("%s: %s" % (name, line.strip()[:120]))
    return found


def test_no_ternary_tower_of_kernel_instances():
    found = ternary_towers()
    assert not found, "pick the instance with by_flags / by_value (launch.cuh):\n" + "\n".join(found)


def test_no_switch_or_macro_per_instance():
    found = case_dispatch()
    assert not found, "pick the instance with by_value (launch.cuh):\n" + "\n".join(found)


def test_the_scan_sees_the_kernels():
    """the checks above would pass vacuously if the kernel scan found nothing, or if the helpers moved"""
    kernels = _global_templates()
    for k in ("fm_backward_kernel", "fm_fused_kernel", "ffm_fused_kernel", "ffm_warp_kernel", "apply_kernel",
              "nfm_mlp_umma_kernel", "key_init_kernel", "csc_backward_long_kernel"):
        assert k in kernels, k
    launch = dict(_sources())["launch.cuh"]
    assert re.search(r"\bauto by_flags\(", launch) and re.search(r"\bauto by_value\(", launch)
