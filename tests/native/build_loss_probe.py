"""Builds tests/native/libhvn_loss_probe.so: the test-only entry point of loss_probe.cu, linked statically
against the object hover_net_b200/build.py produces for the loss kernels (build/loss.o).  Cross-compiles
for sm_90a without a GPU.  Run hover_net_b200.build first."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(ROOT, "hover_net_b200")
SRC = os.path.join(HERE, "loss_probe.cu")
LIB = os.path.join(HERE, "libhvn_loss_probe.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def build(objdir=None, out=LIB, verbose=False):
    """objdir: where loss.o lives (default: the package's build directory)."""
    objdir = objdir or os.path.join(PKG, "build")
    obj = os.path.join(objdir, "loss.o")
    if not os.path.exists(obj):
        raise RuntimeError("%s is missing: build hover_net_b200 first" % obj)
    headers = [os.path.join(PKG, "csrc", f) for f in os.listdir(os.path.join(PKG, "csrc")) if f.endswith((".h", ".cuh"))]
    if os.path.exists(out) and all(os.path.getmtime(out) > os.path.getmtime(d) for d in [obj, SRC] + headers):
        return out
    cmd = [NVCC] + ARCH + ["-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", SRC, obj, "-lcudart", "-o", out]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    print(build(verbose=True))
