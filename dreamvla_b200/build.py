"""Builds libdvla_sm90.so (hand-written CUDA for sm_90a, NVIDIA H100) in-tree with nvcc.

`python -m dreamvla_b200.build` or `__graft_entry__.build()`.  The .so lands in dreamvla_b200/lib/ (git-ignored), where
dreamvla_b200/_lib.py loads it from; nothing is compiled at run time.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libdvla_sm90.so")
SOURCES = ["gemm_sm90.cu", "attention.cu", "attention_small.cu", "norm_act.cu", "loss_optim.cu", "dit_sampler.cu", "augment.cu", "state.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    # host code keeps separate multiplies and adds (no FMA contraction): dvla_bicubic_coeffs must round like Pillow's C
    "-Xcompiler", "-ffp-contract=off",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    return "nvcc"


def _deps_mtime() -> float:
    paths = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "dvla.h")]
    return max(os.path.getmtime(p) for p in paths if os.path.exists(p))


def build_library(force: bool = False, verbose: bool = True) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    if not force and os.path.exists(LIB) and os.path.getmtime(LIB) >= _deps_mtime():
        return LIB
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()

    def compile_one(src: str) -> str:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=len(SOURCES)) as ex:
        objs = list(ex.map(compile_one, SOURCES))
    tmp = LIB + ".tmp"          # link beside the target, then rename: a reader never sees a half-written library
    cmd = [nvcc, "-shared", "-o", tmp, *objs, "-gencode", "arch=compute_90a,code=sm_90a"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    os.replace(tmp, LIB)
    if verbose:
        print(f"[dreamvla_b200.build] built {LIB}", file=sys.stderr)
    return LIB


if __name__ == "__main__":
    build_library(force="--force" in sys.argv)
