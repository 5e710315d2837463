"""Builds libaloam_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

-fmad=false everywhere: float32 results must match an x86-64 (no-FMA) build of the reference bit for bit.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
SO = os.path.join(HERE, "libaloam_b200.so")
SOURCES = ["features.cu", "odometry.cu", "lm.cu", "mapping.cu", "comm.cu", "voxel.cu", "cubemap.cu", "capi.cu", "io.cu"]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
              "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
# float32 decision kernels must not contract a*b+c (bit parity with an x86-64 no-FMA build of the reference);
# lm.cu is double precision, compared at 1e-9, and keeps FMA.
FMAD = {"lm.cu": "-fmad=true"}


def build(force=False, verbose=False):
    srcs = [os.path.join(CSRC, s) for s in SOURCES]
    deps = srcs + [os.path.join(CSRC, h) for h in os.listdir(CSRC) if h.endswith((".h", ".cuh", ".inc"))]
    deps.append(os.path.join(HERE, "..", "include", "aloam_b200.h"))
    deps.append(os.path.join(HERE, "..", "include", "aloam_io.h"))
    if not force and os.path.exists(SO) and all(os.path.getmtime(d) <= os.path.getmtime(SO) for d in deps):
        return SO
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    for s in srcs:
        o = s[:-3] + ".o"
        cmd = [nvcc] + NVCC_FLAGS + [FMAD.get(os.path.basename(s), "-fmad=false"), "-c", s, "-o", o]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if verbose or r.returncode != 0:
            sys.stderr.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed on " + s)
        objs.append(o)
    cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", SO] + objs
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        sys.stderr.write(r.stdout + r.stderr)
        raise RuntimeError("link failed")
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
