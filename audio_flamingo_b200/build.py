"""In-tree nvcc build of libaf3b200.so for sm_90a (cross-compiles without a GPU).

The shared library links against cudart only; the TMA descriptor encoder is fetched from the driver at run time
(cudaGetDriverEntryPoint), so nothing here needs libcuda at build time.  Objects are cached by source mtime and compiler flags.
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
BUILD = PKG_DIR / "_build"
LIB = PKG_DIR / "libaf3b200.so"

SOURCES = [
    "common.cu",
    "gemm_wgmma.cu",
    "attention_wgmma.cu",
    "decode_attention.cu",
    "elementwise.cu",
    "logmel.cu",
    "af3_abi.cu",
]

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
    raise RuntimeError("nvcc not found (needed to build libaf3b200.so)")


def _headers_mtime() -> float:
    hs = list(CSRC.glob("*.h")) + list(CSRC.glob("*.cuh")) + [PKG_DIR.parent / "include" / "af3b200.h"]
    return max(h.stat().st_mtime for h in hs)


def build(force: bool = False, verbose: bool = False) -> Path:
    nvcc = _nvcc()
    BUILD.mkdir(exist_ok=True)
    hm = _headers_mtime()
    # objects built with other flags (another architecture, say) are never reused: the flags are part of the cache key
    stamp = BUILD / "flags.txt"
    flags = " ".join([nvcc, *NVCC_FLAGS])
    if not stamp.exists() or stamp.read_text() != flags:
        force = True
    jobs = []
    objs = []
    for src in SOURCES:
        s = CSRC / src
        o = BUILD / (s.stem + ".o")
        objs.append(o)
        if force or not o.exists() or o.stat().st_mtime < max(s.stat().st_mtime, hm):
            jobs.append([nvcc, *NVCC_FLAGS, "-c", str(s), "-o", str(o)])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed: {' '.join(cmd)}\n{r.stdout}\n{r.stderr}")

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(run, jobs))
    if jobs or not LIB.exists():
        run([nvcc, "-shared", "-cudart", "static", "-o", str(LIB), *map(str, objs)])
    stamp.write_text(flags)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
