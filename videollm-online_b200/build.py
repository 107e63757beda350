"""In-tree build of libvlo_b200.so (hand-written sm_90a CUDA for the H100 behind a C ABI).

nvcc cross-compiles for sm_90a without a GPU, so the library can be built on a machine
without one; the resulting .so is git-ignored.  Builds nothing else: the oracle is pure
Python/torch.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import pathlib
import shutil
import subprocess
import sys

PKG = pathlib.Path(__file__).resolve().parent
CSRC = PKG / "csrc"
OBJ = PKG / "build"
LIB = PKG / "libvlo_b200.so"
INCLUDE = PKG.parent / "include"

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
    "-cudart", "static",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _stale(target: pathlib.Path, deps: list[pathlib.Path]) -> bool:
    if not target.exists():
        return True
    t = target.stat().st_mtime
    return any(d.stat().st_mtime > t for d in deps)


def build(force: bool = False, verbose: bool = False, debug: bool = False) -> pathlib.Path:
    """debug=True: a second library (libvlo_b200_dbg.so, objects in build_dbg/) whose bounded mbarrier waits trap after
    2^16 polls instead of 2^24 and print the stuck (block, thread) first, so a protocol dead-lock is reported within
    seconds; select it with VLO_LIB=.../libvlo_b200_dbg.so."""
    global OBJ, LIB
    nvcc = _nvcc()
    flags_extra = []
    if debug:
        OBJ, LIB = PKG / "build_dbg", PKG / "libvlo_b200_dbg.so"
        flags_extra = ["-DVLO_MBAR_BOUND_LOG2=16", "-DVLO_MBAR_TRACE=1"]
    OBJ.mkdir(exist_ok=True)
    headers = sorted(CSRC.glob("*.cuh")) + sorted(CSRC.glob("*.h")) + sorted(INCLUDE.glob("*.h"))
    sources = sorted(CSRC.glob("*.cu"))
    jobs = []
    objs = []
    for src in sources:
        obj = OBJ / (src.stem + ".o")
        objs.append(obj)
        if force or _stale(obj, [src, *headers, pathlib.Path(__file__)]):
            jobs.append([nvcc, *NVCC_FLAGS, *flags_extra, "-I", str(INCLUDE), "-I", str(CSRC), "-c", str(src), "-o", str(obj)])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            sys.stderr.write(r.stdout + r.stderr)

    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(run, jobs))
    if jobs or force or _stale(LIB, objs):
        run([nvcc, "-shared", *NVCC_FLAGS, "-o", str(LIB), *map(str, objs)])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, debug="--debug" in sys.argv))
