"""Build libegnn_b200.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m egnn_pytorch_b200.build [--force]
"""
from __future__ import annotations

import glob
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIB_DIR, "libegnn_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
]
OBJ_DIR = os.path.join(HERE, "build")          # git-ignored; objects are rebuilt per source when stale


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def is_stale():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h"))
    return any(os.path.getmtime(p) > t for p in deps)


def _deps():
    return glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.h")) + \
        glob.glob(os.path.join(HERE, "..", "include", "*.h"))


def build(force=False, verbose=False):
    """One nvcc process per translation unit (run concurrently), then one link step."""
    if not force and not is_stale():
        return LIB
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: cannot build libegnn_b200.so")
    os.makedirs(LIB_DIR, exist_ok=True)
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdr_time = max([os.path.getmtime(p) for p in _deps()] + [0.0])
    jobs, objs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if not force and os.path.exists(obj) and os.path.getmtime(obj) > max(os.path.getmtime(src), hdr_time):
            continue
        cmd = [nvcc] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", "-o", obj, src]
        jobs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True)))
    failed = False
    for src, proc in jobs:
        out, err = proc.communicate()
        if proc.returncode != 0:
            sys.stderr.write(out + err)
            failed = True
        elif verbose:
            sys.stderr.write(err)
    if failed:
        raise RuntimeError("nvcc failed building libegnn_b200.so")
    cmd = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-Xcompiler", "-fPIC", "-lcuda", "-o", LIB] + objs
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
        raise RuntimeError("nvcc failed linking libegnn_b200.so")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
