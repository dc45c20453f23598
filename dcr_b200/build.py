"""In-tree build of libdcr_b200.so (sm_90a, NVIDIA H100).

`python -m dcr_b200.build` or `__graft_entry__.build()`.  nvcc cross-compiles without a GPU.  Objects are cached by
source mtime so a rebuild after touching one .cu file takes seconds.
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
BUILD_DIR = PKG_DIR / "_build"
LIB_PATH = PKG_DIR / "libdcr_b200.so"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and Path(cand).exists():
            return cand
    raise RuntimeError("nvcc not found (set NVCC=/path/to/nvcc)")


def _needs(obj: Path, deps: list[Path]) -> bool:
    if not obj.exists():
        return True
    t = obj.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def build(verbose: bool = False, force: bool = False) -> Path:
    nvcc = _nvcc()
    BUILD_DIR.mkdir(exist_ok=True)
    sources = sorted(CSRC.glob("*.cu"))
    headers = sorted(CSRC.glob("*.cuh")) + [PKG_DIR.parent / "include" / "dcr_b200.h", Path(__file__)]
    jobs = []
    objs = []
    for src in sources:
        obj = BUILD_DIR / (src.stem + ".o")
        objs.append(obj)
        if force or _needs(obj, [src] + headers):
            jobs.append([nvcc, *NVCC_FLAGS, "-c", str(src), "-o", str(obj)])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"build failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")
        return r

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    if jobs or force or _needs(LIB_PATH, objs):
        # cudart linked statically: the .so only needs libcuda (driver) at run time, resolved lazily by cudart
        run([nvcc, "-shared", "-o", str(LIB_PATH), *map(str, objs), "-cudart", "static",
             "-gencode", "arch=compute_90a,code=sm_90a"])
    return LIB_PATH


if __name__ == "__main__":
    p = build(verbose=True, force="--force" in sys.argv)
    print(p)
