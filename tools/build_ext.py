"""In-tree build of the native extensions.

* ``sparkflow_b200/_C.so``    – sm_90a kernels (csrc/kernels.cu) + host runtime (csrc/runtime.cpp)
* ``sparkflow_b200/_host.so`` – CPU-only native helpers (TF bundle codec, crc32c, carrier codec, CSV)

nvcc cross-compiles for sm_90a without a GPU; the resulting ``.so`` files are git-ignored.  Objects are cached by
source hash under ``build/``.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
import sysconfig
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
CSRC = ROOT / "csrc"
BUILD = ROOT / "build"
PKG = ROOT / "sparkflow_b200"

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
CXX = os.environ.get("CXX") or shutil.which("g++") or "g++"
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]


def _includes() -> list[str]:
    import pybind11

    return [
        f"-I{pybind11.get_include()}",
        f"-I{sysconfig.get_paths()['include']}",
        f"-I{CSRC}",
        "-I/usr/local/cuda/include",
    ]


def _digest(paths: list[Path], extra: str) -> str:
    h = hashlib.sha256(extra.encode())
    for p in sorted(paths):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    return h.hexdigest()[:16]


def _run(cmd: list[str]) -> None:
    proc = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if proc.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + proc.stdout + "\n")
        raise RuntimeError(f"build step failed: {cmd[0]} (exit {proc.returncode})")
    if os.environ.get("SPARKFLOW_BUILD_VERBOSE"):
        sys.stderr.write(proc.stdout)


def _compile_cuda(verbose_ptxas: bool) -> Path:
    srcs = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [CSRC / "sf_api.h"]
    flags = ARCH_FLAGS + ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]
    if verbose_ptxas:
        flags += ["-Xptxas", "-v"]
    tag = _digest(srcs, " ".join(flags))
    obj = BUILD / f"kernels.{tag}.o"
    if not obj.exists():
        _run([NVCC, *flags, f"-I{CSRC}", "-c", str(CSRC / "kernels.cu"), "-o", str(obj)])
    return obj


def _compile_cxx(name: str, deps: list[Path]) -> Path:
    flags = ["-O2", "-std=c++17", "-fPIC", "-fvisibility=hidden", "-Wall", "-Wno-unused-function"]
    tag = _digest(deps, " ".join(flags))
    obj = BUILD / f"{name}.{tag}.o"
    if not obj.exists():
        _run([CXX, *flags, *_includes(), "-c", str(CSRC / f"{name}.cpp"), "-o", str(obj)])
    return obj


def build(verbose_ptxas: bool = False, only: str | None = None) -> dict[str, Path]:
    BUILD.mkdir(exist_ok=True)
    out: dict[str, Path] = {}
    jobs = {}
    with ThreadPoolExecutor(max_workers=4) as ex:
        if only in (None, "cuda"):
            jobs["kernels"] = ex.submit(_compile_cuda, verbose_ptxas)
            jobs["runtime"] = ex.submit(_compile_cxx, "runtime", [CSRC / "runtime.cpp", CSRC / "sf_api.h", CSRC / "vmm.h"])
        if only in (None, "host") and (CSRC / "hostlib.cpp").exists():
            jobs["hostlib"] = ex.submit(_compile_cxx, "hostlib", [CSRC / "hostlib.cpp"])
        objs = {k: f.result() for k, f in jobs.items()}
    # keep only the objects just used: stale ones would otherwise pile up under build/
    for k, keep in objs.items():
        for old in BUILD.glob(f"{k}.*.o"):
            if old != keep:
                old.unlink()

    if "kernels" in objs:
        so = PKG / "_C.so"
        _run([
            NVCC, "-shared", *ARCH_FLAGS, "-Xcompiler", "-fPIC", str(objs["kernels"]), str(objs["runtime"]),
            "-o", str(so), "-cudart", "static", "-lcuda" if os.environ.get("SPARKFLOW_LINK_LIBCUDA") else "-ldl",
        ])
        out["_C"] = so
    if "hostlib" in objs:
        so = PKG / "_host.so"
        _run([CXX, "-shared", "-fPIC", str(objs["hostlib"]), "-o", str(so)])
        out["_host"] = so
    return out


if __name__ == "__main__":
    res = build(verbose_ptxas="-v" in sys.argv)
    for k, v in res.items():
        print(f"built {k}: {v} ({v.stat().st_size/1024:.0f} KiB)")
