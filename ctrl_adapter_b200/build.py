"""In-tree build of libctrl_adapter_b200.so: nvcc cross-compiles every .cu for sm_90a (works without a GPU)."""
from __future__ import annotations

import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libctrl_adapter_b200.so")
SOURCES = ["gemm_conv.cu", "gemm_conv_bn64.cu", "gemm_conv_bn128.cu", "gemm_conv_bn160.cu", "gemm_conv_bn256.cu",
           "attention.cu", "temporal_attention.cu", "norm.cu", "elementwise.cu", "capi.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]


def _newer(target: str, deps) -> bool:
    if not os.path.exists(target):
        return False
    t = os.path.getmtime(target)
    return all(os.path.getmtime(d) <= t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(BUILD, exist_ok=True)
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "ctrl_adapter_b200.h"))
    objs, jobs = [], []
    for src in SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src.replace(".cu", ".o"))
        objs.append(o)
        if force or not _newer(o, [s] + headers):
            jobs.append([NVCC] + FLAGS + ["-c", s, "-o", o])

    def run(cmd):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed: " + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        if verbose and (r.stdout or r.stderr):
            sys.stderr.write(r.stdout + r.stderr)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(len(jobs), os.cpu_count() or 4)) as ex:
            list(ex.map(run, jobs))
    if jobs or force or not _newer(LIB, objs):
        run([NVCC, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-o", LIB] + objs)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
