"""Build the CPU-emulated kernel library (TEST INFRASTRUCTURE, see cuda_emu.h):
the .cu sources of gcc_b200/csrc compiled by g++ with -DGCCB_EMU.  Only the
`-m "not gpu"` kernel-logic tests load it; the product never does."""
import glob
import os
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
CSRC = os.path.join(ROOT, "gcc_b200", "csrc")
OUT = os.path.join(HERE, "_build")
LIB = os.path.join(OUT, "libgccb200_emu.so")
# kernels that need real sm_90a hardware features (wgmma/TMA) are excluded
EXCLUDE = {"tc_gemm.cu"}


def sources():
    return sorted(f for f in glob.glob(os.path.join(CSRC, "*.cu"))
                  if os.path.basename(f) not in EXCLUDE)


def build(force=False):
    os.makedirs(OUT, exist_ok=True)
    hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + \
        [os.path.join(HERE, "cuda_emu.h"), os.path.join(ROOT, "include", "gccb200.h")]
    objs, relink = [], force or not os.path.exists(LIB)
    for src in sources():
        obj = os.path.join(OUT, os.path.basename(src) + ".o")
        if force or not os.path.exists(obj) or any(
                os.path.getmtime(obj) < os.path.getmtime(d) for d in [src] + hdrs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-DGCCB_EMU", "-DGCCB_HUB_DEG=3", "-I", HERE,
                                   "-x", "c++", "-c", src, "-o", obj])
            relink = True
        objs.append(obj)
    if relink:
        subprocess.check_call(["g++", "-shared", "-o", LIB] + objs)
    return LIB


if __name__ == "__main__":
    print(build(force=True))
