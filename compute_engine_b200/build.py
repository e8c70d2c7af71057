"""In-tree build of the native pieces (no JIT cache: the built .so files travel to
the GPU box with the gpurun snapshot).

  liblce_b200.so        CUDA kernels + C-ABI (nvcc, sm_90a only)
  liblce_b200_host.so   C++ TFLite-custom-op shell / graph host above the C-ABI
"""
from __future__ import annotations

import os
import shutil
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
INC = os.path.join(REPO, "include")

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo",
              "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]


def _newer(target, sources):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in sources)


def _nvcc():
    return shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"


def cuda_lib_path():
    return os.path.join(PKG, "liblce_b200.so")


def host_lib_path():
    return os.path.join(PKG, "liblce_b200_host.so")


def build_cuda(force=False, verbose=False):
    out = cuda_lib_path()
    srcs = [os.path.join(CSRC, f) for f in os.listdir(CSRC)
            if f.endswith((".cu", ".cuh"))] + \
           [os.path.join(INC, f) for f in os.listdir(INC)]
    if not force and not _newer(out, srcs):
        return out
    cus = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))
    cmd = [_nvcc(), *NVCC_FLAGS, "-I", INC, *cus, "-o", out]
    if os.environ.get("LCE_TC_PROF_BUILD") == "1":      # development: per-role cycle counters
        cmd.insert(1, "-DLCE_TC_PROF=1")
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    subprocess.run(cmd, check=True)
    return out


def build_host(force=False):
    hdir = os.path.join(CSRC, "host")
    if not os.path.isdir(hdir):
        return None
    out = host_lib_path()
    ccs = sorted(os.path.join(hdir, f) for f in os.listdir(hdir) if f.endswith(".cc"))
    hs = [os.path.join(hdir, f) for f in os.listdir(hdir) if f.endswith(".h")] + \
         [os.path.join(INC, f) for f in os.listdir(INC)]
    if not ccs:
        return None
    if not force and not _newer(out, ccs + hs + [cuda_lib_path()]):
        return out
    cuda_home = os.path.dirname(os.path.dirname(_nvcc()))
    cmd = ["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-Wall", "-I", INC, "-I", hdir,
           "-I", os.path.join(cuda_home, "include"), *ccs, "-o", out,
           "-L", PKG, "-l:liblce_b200.so", "-Wl,-rpath,$ORIGIN",
           "-L", os.path.join(cuda_home, "lib64"), "-lcudart_static", "-ldl", "-lrt",
           "-pthread"]
    subprocess.run(cmd, check=True)
    return out


def build_all(force=False):
    build_cuda(force)
    build_host(force)


if __name__ == "__main__":
    import sys
    build_all(force="--force" in sys.argv)
    print("built", cuda_lib_path())
