"""Builds libb200zk.so (the C-ABI shared library) in-tree with nvcc for sm_90a (H100).

    python scroll-prover_b200/build.py [--force]

The .so and the object files are build products (git-ignored); build() rebuilds whatever is missing or stale.
"""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_obj")
LIB = os.path.join(HERE, "libb200zk.so")
SOURCES = ["api.cu", "ntt.cu", "msm.cu", "poly.cu", "g1fft.cu", "quotient.cu", "lookup.cu", "mock.cu", "comm.cu"]
HEADERS = ["ff.cuh", "ec.cuh", "common.cuh", os.path.join("..", "..", "include", "b200zk.h"), "graph.hpp", "graph_exec.cuh", "lookup.cuh"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]  # H100: the one architecture the library is built for
FLAGS = GENCODE + [ "-O3", "-std=c++17", "-lineinfo",
         "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _stale(target: str, deps: list[str]) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    jobs = []
    for s in SOURCES:
        src = os.path.join(CSRC, s)
        obj = os.path.join(OBJ, s.replace(".cu", ".o"))
        if force or _stale(obj, [src] + hdrs):
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            jobs.append(cmd)

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: %s\n%s\n%s" % (" ".join(cmd), r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)

    with ThreadPoolExecutor(max_workers=4) as ex:
        list(ex.map(run, jobs))
    objs = [os.path.join(OBJ, s.replace(".cu", ".o")) for s in SOURCES]
    if force or jobs or _stale(LIB, objs):
        cmd = [NVCC, "-shared", "-o", LIB] + objs + GENCODE + ["-ldl"]
        run(cmd)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
