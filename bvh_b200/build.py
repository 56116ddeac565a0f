"""bvh_b200/build.py -- compiles the CUDA sources into bvh_b200/libbvh_b200.so (sm_90a only).

    python -m bvh_b200.build [--force] [--ptxas-v]

nvcc cross-compiles without a GPU.  Flags that matter:
  -gencode arch=compute_90a,code=sm_90a     H100 only, no PTX fallback for other architectures
  -fmad=false                               no FMA contraction: bit parity with the reference (DESIGN.md)
  -lineinfo                                 ncu source view
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "build")
SO = os.path.join(HERE, "libbvh_b200.so")
SOURCES = ["capi.cu", "build_sah.cu", "flatten.cu", "traverse.cu", "lbvh.cu", "closest.cu", "dim2.cu", "dynamic.cu", "dim4.cu", "tripairs.cu", "segments.cu"]
HEADERS = ["common.cuh", "internal.h", "build_types.cuh", "csr.cuh", "queries.cuh", "update.cuh", "dynamic.cuh", "tritri.cuh", "exact.cuh", os.path.join("..", "..", "include", "bvh_b200.h")]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo", "-fmad=false",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
    "-Xcudafe", "--diag_suppress=177", "-Xcudafe", "--diag_suppress=550",
]


def _stale(target: str, deps) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False, ptxas_v: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    srcs = [s for s in SOURCES if os.path.exists(os.path.join(CSRC, s))]
    hdrs = [os.path.join(CSRC, h) for h in HEADERS] + [os.path.abspath(__file__)]
    jobs = []
    for s in srcs:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if ptxas_v else []) + ["-c", src, "-o", obj]
            jobs.append(cmd)
    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        return cmd, r
    if jobs:
        with ThreadPoolExecutor(max_workers=min(6, len(jobs))) as ex:
            for cmd, r in ex.map(run, jobs):
                if verbose or ptxas_v or r.returncode != 0:
                    sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + r.stderr)
                if r.returncode != 0:
                    raise RuntimeError("nvcc failed for " + cmd[-3])
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in srcs]
    if force or jobs or _stale(SO, objs):
        cmd = [NVCC, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-Xcompiler", "-fPIC", "-o", SO] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
            raise RuntimeError("link failed")
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True, ptxas_v="--ptxas-v" in sys.argv))
