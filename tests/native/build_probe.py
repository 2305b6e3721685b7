"""Builds tests/native/libhvn_probe.so: the test-only operator entry points of conv_probe.cu, linked statically against
the kernel objects hover_net_b200/build.py produces (build/conv_tc.o, build/conv_ref.o).  Cross-compiles for sm_90a
without a GPU.  Run hover_net_b200.build first."""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
PKG = os.path.join(ROOT, "hover_net_b200")
SRC = os.path.join(HERE, "conv_probe.cu")
LIB = os.path.join(HERE, "libhvn_probe.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]


def build(objdir=None, out=LIB, verbose=False):
    """objdir: where conv_tc.o / conv_ref.o live (default: the package's build directory)."""
    objdir = objdir or os.path.join(PKG, "build")
    objs = [os.path.join(objdir, o) for o in ("conv_tc.o", "conv_ref.o")]
    for o in objs:
        if not os.path.exists(o):
            raise RuntimeError("%s is missing: build hover_net_b200 first" % o)
    headers = [os.path.join(PKG, "csrc", f) for f in os.listdir(os.path.join(PKG, "csrc")) if f.endswith((".h", ".cuh"))]
    if os.path.exists(out) and all(os.path.getmtime(out) > os.path.getmtime(d) for d in objs + headers + [SRC]):
        return out
    cmd = [NVCC] + ARCH + ["-O2", "-std=c++17", "-Xcompiler", "-fPIC", "-shared", SRC] + objs + ["-lcudart", "-o", out]
    if verbose:
        print(" ".join(cmd))
    subprocess.check_call(cmd)
    return out


if __name__ == "__main__":
    print(build(verbose=True))
