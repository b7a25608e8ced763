"""Build libfastfp_b200.so in-tree with nvcc for sm_90a (H100) (no torch, no cmake).

``python -m fastfp_b200.build`` or ``__graft_entry__.build()``. nvcc cross-compiles without a
GPU. The library links cudart statically, so it only needs the driver at run time.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
OUT_DIR = os.path.join(HERE, "_lib")
LIB = os.path.join(OUT_DIR, "libfastfp_b200.so")
SOURCES = ["cabi.cu", "precompute.cu", "fp_sweep.cu", "fp_sweep_w1.cu", "fp_sweep_w2.cu", "fp_sweep_w4.cu",
           "fp_sweep_wide.cu", "fp_sweep_xwide.cu", "fp_sweep_i8.cu", "fe.cu", "nmfp.cu", "xcy.cu", "microbench.cu", "hostutil.cu",
           "sim.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-fmad=true"]
# developer builds only (e.g. FASTFP_B200_NVCC_FLAGS=-DFFP_DEBUG_SWITCHES for tools/dbg_split.sh); the
# shipped library is built without it and bench.py refuses to run a library built with extra flags
EXTRA = os.environ.get("FASTFP_B200_NVCC_FLAGS", "").split()


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def _digest() -> str:
    h = hashlib.sha256()
    for name in sorted(os.listdir(CSRC)) + ["../../include/fastfp_b200.h"]:
        path = os.path.join(CSRC, name)
        if os.path.isfile(path):
            with open(path, "rb") as f:
                h.update(name.encode() + b"\0" + f.read())
    h.update(" ".join(ARCH + FLAGS + EXTRA).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    stamp = os.path.join(OUT_DIR, "build.sha256")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    nvcc = _nvcc()
    objs = [os.path.join(OUT_DIR, s.replace(".cu", ".o")) for s in SOURCES]

    def compile_one(pair):
        src, obj = pair
        cmd = [nvcc, *ARCH, *FLAGS, *EXTRA, "-I", INCLUDE, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return src, r.stderr

    with ThreadPoolExecutor(max_workers=min(len(SOURCES), os.cpu_count() or 4)) as ex:
        logs = list(ex.map(compile_one, zip(SOURCES, objs)))
    if verbose:
        for src, log in logs:
            print(f"==== {src}\n{log}")
    cmd = [nvcc, *ARCH, "-shared", "-cudart", "static", "-o", LIB, *objs]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
