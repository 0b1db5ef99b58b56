"""Per-kernel resource usage of the built kernel library, read without a GPU: `cuobjdump -res-usage` on
sparkflow_b200/_C.so, with the names demangled by `c++filt`."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SO = os.path.join(ROOT, "sparkflow_b200", "_C.so")

# a test that reads the built library needs it and the CUDA binary utilities
needs_binary_utils = pytest.mark.skipif(
    not os.path.exists(SO) or shutil.which("cuobjdump") is None or shutil.which("c++filt") is None,
    reason="needs the built extension and the CUDA binary utilities")


def res_usage():
    """{kernel name, demangled, without its parameter list (e.g. ``sf::sf_gemm_kernel<32, false, 0, false, false>``):
    (registers, stack frame bytes)}"""
    txt = subprocess.run(["cuobjdump", "-res-usage", SO], stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, check=True).stdout
    names = re.findall(r"Function (\S+):\n\s+REG:(\d+) STACK:(\d+)", txt)
    dem = subprocess.run(["c++filt"], input="\n".join(n for n, _, _ in names), stdout=subprocess.PIPE, text=True, check=True).stdout.splitlines()
    return {re.sub(r"\(.*", "", d).replace("void ", ""): (int(r), int(s)) for d, (_, r, s) in zip(dem, names)}


def gemm_instances(use):
    """The one-CTA GEMM kernel instances in ``use`` (a res_usage() result): {(BN, MN, EPI, EXT, PEN): (registers, stack
    frame bytes)}, EPI an SfEpi value (csrc/sf_api.h)"""
    out = {}
    for k, v in use.items():
        m = re.fullmatch(r"sf::sf_gemm_kernel<(\d+), (false|true), (\d+), (false|true), (false|true)>", k)
        if m:
            out[(int(m[1]), m[2] == "true", int(m[3]), m[4] == "true", m[5] == "true")] = v
    return out
