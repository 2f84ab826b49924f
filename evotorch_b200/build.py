"""Build libevok.so (the C-ABI library of sm_90a kernels) in-tree with nvcc.

    python -m evotorch_b200.build [--force] [--verbose]

The library is written to evotorch_b200/lib/libevok.so (git-ignored build product).  nvcc cross-compiles for sm_90a
without a GPU.
"""

from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG, "csrc")
LIBDIR = os.path.join(PKG, "lib")
LIB = os.path.join(LIBDIR, "libevok.so")
OBJDIR = os.path.join(PKG, "build", "obj")

NVCC_FLAGS = [
    "-O3",
    "-std=c++17",
    "-gencode",
    "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler",
    "-fPIC",
    "-Xcompiler",
    "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def sources() -> list:
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newest_input() -> float:
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(PKG, "..", "include", "evok.h"), __file__]
    return max(os.path.getmtime(p) for p in deps)


def is_up_to_date() -> bool:
    return os.path.exists(LIB) and os.path.getmtime(LIB) >= _newest_input()


def build(force: bool = False, verbose: bool = False, defines: tuple = (), tag: str = "") -> str:
    """Build libevok.so.  `defines` / `tag` build a tuning variant lib/libevok_<tag>.so (used by scripts/kbench.py)."""
    global OBJDIR
    lib_path = LIB if not tag else os.path.join(LIBDIR, f"libevok_{tag}.so")
    if not tag and not force and is_up_to_date():
        return LIB
    nvcc = _nvcc()
    objdir = OBJDIR if not tag else os.path.join(PKG, "build", f"obj_{tag}")
    os.makedirs(objdir, exist_ok=True)
    os.makedirs(LIBDIR, exist_ok=True)
    extra = (["-Xptxas", "-v"] if verbose else []) + [f"-D{d}" for d in defines]

    def compile_one(src: str) -> str:
        obj = os.path.join(objdir, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(sources()))) as ex:
        objs = list(ex.map(compile_one, sources()))
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-o", lib_path + ".tmp", *objs,
           "-lcuda"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
        raise RuntimeError("link failed")
    os.replace(lib_path + ".tmp", lib_path)
    return lib_path


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
