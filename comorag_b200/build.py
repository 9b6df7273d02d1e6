"""Build recipe for libcomorag_b200.so (hand-written sm_90a CUDA, C ABI).

nvcc cross-compiles for sm_90a without a GPU, so the library can be built on a
machine without one; the resulting .so is git-ignored.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_DIR = PKG_DIR / "lib"
LIB_PATH = LIB_DIR / "libcomorag_b200.so"
INCLUDE = PKG_DIR.parent / "include"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--shared", "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
]


LAST_BUILD_MODE = "not built in this process"


def _nvcc() -> str:
    exe = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(exe):
        raise RuntimeError("nvcc not found; cannot build libcomorag_b200.so")
    return exe


def sources() -> list[Path]:
    return sorted(CSRC.glob("*.cu"))


def _stale() -> bool:
    if not LIB_PATH.exists():
        return True
    built = LIB_PATH.stat().st_mtime
    deps = list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + list(INCLUDE.glob("*.h")) + [Path(__file__)]
    return any(p.stat().st_mtime > built for p in deps)


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every csrc/*.cu into one shared library; returns its path."""
    global LAST_BUILD_MODE
    if not force and not _stale():
        LAST_BUILD_MODE = "up-to-date (every csrc/*.cu, *.cuh and include/*.h is older than the .so)"
        return LIB_PATH
    LAST_BUILD_MODE = "compiled with nvcc -gencode arch=compute_90a,code=sm_90a"
    LIB_DIR.mkdir(parents=True, exist_ok=True)
    objs = []
    obj_dir = LIB_DIR / "obj"
    obj_dir.mkdir(exist_ok=True)
    procs = []
    flags = [f for f in NVCC_FLAGS if f != "--shared"]
    for src in sources():
        obj = obj_dir / (src.stem + ".o")
        objs.append(obj)
        cmd = [_nvcc(), *flags, "-I", str(INCLUDE), "-c", str(src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(f"--- nvcc {src.name} (rc={p.returncode})\n{out}\n")
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed; see output above")
    tmp = LIB_PATH.with_suffix(".so.tmp")
    link = [_nvcc(), "--shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", str(tmp), *map(str, objs)]
    subprocess.run(link, check=True)
    os.replace(tmp, LIB_PATH)
    return LIB_PATH


EXAMPLES = PKG_DIR.parent / "examples"
EXAMPLE_BIN = EXAMPLES / "bin" / "c_host_search"


def build_examples(force: bool = False) -> Path:
    """examples/c_host_search.cu -> examples/bin/c_host_search: a host with no torch / Python in it, linked against the
    C ABI only (rpath relative to the binary, so it runs wherever the repo snapshot lands)."""
    src = EXAMPLES / "c_host_search.cu"
    deps = [src, LIB_PATH, *INCLUDE.glob("*.h")]
    if not force and EXAMPLE_BIN.exists() and all(p.stat().st_mtime <= EXAMPLE_BIN.stat().st_mtime for p in deps):
        return EXAMPLE_BIN
    EXAMPLE_BIN.parent.mkdir(parents=True, exist_ok=True)
    cmd = [_nvcc(), "-gencode", "arch=compute_90a,code=sm_90a", "-O2", "-std=c++17", "-lineinfo", "-I", str(INCLUDE),
           str(src), "-o", str(EXAMPLE_BIN), "-L", str(LIB_DIR), "-lcomorag_b200",
           "-Xlinker", "-rpath", "-Xlinker", "$ORIGIN/../../comorag_b200/lib"]
    subprocess.run(cmd, check=True)
    return EXAMPLE_BIN


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
