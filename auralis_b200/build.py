"""Builds libxtts_b200.so in-tree with nvcc for sm_90a (no torch in the link line).

`python -m auralis_b200.build` or `build_native()`; nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libxtts_b200.so")
SOURCES = ["engine.cu", "gpt_kernels.cu", "gemm_simt.cu", "gemm_wgmma.cu", "gemm_wgmma_wide.cu", "vocoder.cu", "conv1d_tc.cu", "cond.cu", "enhance.cu", "pvoc.cu", "flac.cu", "resample.cu", "beam.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = [*ARCH, "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xcompiler", "-pthread"]


def _stale() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "xtts_b200.h")]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build_native(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    procs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(HERE, "build", src.replace(".cu", ".o"))
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(
                os.path.getmtime(os.path.join(CSRC, f)) for f in os.listdir(CSRC)):
            continue
        cmd = [nvcc, *NVCC_FLAGS, "-c", sp, "-o", obj]
        if verbose:
            print(" ".join(cmd))
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            sys.stderr.write(out.decode())
            raise RuntimeError(f"nvcc failed on {src}")
        if verbose and out:
            print(out.decode())
    cmd = [nvcc, "-shared", "-o", LIB, *objs, "-Xcompiler", "-pthread", *ARCH]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        sys.stderr.write(r.stdout.decode())
        raise RuntimeError("link failed")
    return LIB


if __name__ == "__main__":
    print(build_native(force="--force" in sys.argv, verbose=True))
