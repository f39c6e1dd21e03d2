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
# The default build routes every row with more than 3 neighbours to the CTA-wide hub gathers, so that the kernel-logic
# tests reach them on small ego-nets.  hub_deg=None keeps the product's threshold (GCCB_HUB_DEG = 256): the warp
# gathers' unrolled bodies (eight / four neighbours per step) then run too.  Each variant has its own directory.
HUB_DEG_TESTS = 3
# kernels that need real sm_90a hardware features (wgmma/TMA) are excluded
EXCLUDE = {"tc_gemm.cu"}


def sources():
    return sorted(f for f in glob.glob(os.path.join(CSRC, "*.cu"))
                  if os.path.basename(f) not in EXCLUDE)


def build(force=False, hub_deg=HUB_DEG_TESTS):
    out = OUT if hub_deg == HUB_DEG_TESTS else os.path.join(OUT, "hub_deg_default" if hub_deg is None else "hub_deg_%d" % hub_deg)
    lib = LIB if out == OUT else os.path.join(out, "libgccb200_emu.so")
    defs = ["-DGCCB_EMU"] + ([] if hub_deg is None else ["-DGCCB_HUB_DEG=%d" % hub_deg])
    os.makedirs(out, exist_ok=True)
    hdrs = glob.glob(os.path.join(CSRC, "*.cuh")) + \
        [os.path.join(HERE, "cuda_emu.h"), os.path.join(ROOT, "include", "gccb200.h")]
    objs, relink = [], force or not os.path.exists(lib)
    for src in sources():
        obj = os.path.join(out, os.path.basename(src) + ".o")
        if force or not os.path.exists(obj) or any(
                os.path.getmtime(obj) < os.path.getmtime(d) for d in [src] + hdrs):
            subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC"] + defs + ["-I", HERE,
                                   "-x", "c++", "-c", src, "-o", obj])
            relink = True
        objs.append(obj)
    if relink:
        subprocess.check_call(["g++", "-shared", "-o", lib] + objs)
    return lib


if __name__ == "__main__":
    print(build(force=True))
