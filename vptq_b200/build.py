"""Build libvptq_b200.so in-tree with nvcc for sm_90a (H100; no CMake, no pybind, no torch headers).

    python -m vptq_b200.build [--force] [--verbose]

The shared library is written next to this file (vptq_b200/libvptq_b200.so, git-ignored).  nvcc
cross-compiles without a GPU.
"""
from __future__ import annotations

import argparse
import concurrent.futures as cf
import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
OBJ = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libvptq_b200.so")

SOURCES = ["api.cu", "gemv.cu", "gemv_inst_v8.cu", "gemv_inst_vx.cu", "gemv_lists.cu", "gemv_lists_batch.cu", "gemv_lists16.cu", "lists_build.cu", "lists_dense.cu", "dequant.cu", "gemv_v2.cu", "gemm_wgmma.cu", "wgrad.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = (["-DVPTQ_B200_PROF_WARPS"] if os.environ.get("VPTQ_B200_PROF_WARPS") else []) + [*ARCH, "-lineinfo", "-O3", "-std=c++17",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _digest(paths):
    h = hashlib.sha256()
    h.update(" ".join(FLAGS).encode())
    for p in sorted(paths):
        with open(p, "rb") as f:
            h.update(p.encode())
            h.update(f.read())
    return h.hexdigest()


def _headers():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(INCLUDE, "vptq_b200.h"))
    hs.append(os.path.join(INCLUDE, "vptq_b200_grad.h"))
    hs.append(os.path.join(INCLUDE, "vptq_b200_graph.h"))
    hs.append(os.path.join(INCLUDE, "vptq_b200_batch.h"))
    hs.append(os.path.join(INCLUDE, "vptq_b200_lists_dense.h"))
    hs.append(os.path.join(INCLUDE, "vptq_b200_lists16.h"))
    return hs


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdr = _headers()
    objs, jobs = [], []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        stamp = obj + ".sha"
        want = _digest([src] + hdr)
        have = open(stamp).read() if os.path.exists(stamp) else ""
        objs.append(obj)
        if force or have != want or not os.path.exists(obj):
            jobs.append((src, obj, stamp, want))

    def compile_one(job):
        src, obj, stamp, want = job
        cmd = [NVCC, *FLAGS, "-I", INCLUDE, "-c", src, "-o", obj]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        with open(stamp, "w") as f:
            f.write(want)
        return obj

    if jobs:
        with cf.ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or not os.path.exists(LIB):
        cmd = [NVCC, "-shared", "-o", LIB, *objs, *ARCH,
               "-Xcompiler", "-fPIC", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
