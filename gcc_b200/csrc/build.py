"""Build libgccb200.so (hand-written sm_90a CUDA + the C ABI) with nvcc, in-tree.

    python -m gcc_b200.csrc.build          # or: __graft_entry__.build()

nvcc cross-compiles without a GPU.  The library lands next to the package
(gcc_b200/libgccb200.so, git-ignored), objects under gcc_b200/build/.
"""
import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
PKG = os.path.dirname(HERE)
ROOT = os.path.dirname(PKG)
LIB = os.path.join(PKG, "libgccb200.so")
OBJ_DIR = os.path.join(PKG, "build")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def sources():
    return sorted(glob.glob(os.path.join(HERE, "*.cu")))


def _stale(target, deps):
    return not os.path.exists(target) or any(os.path.getmtime(d) > os.path.getmtime(target) for d in deps)


def build(force=False, verbose=False):
    os.makedirs(OBJ_DIR, exist_ok=True)
    hdrs = glob.glob(os.path.join(HERE, "*.cuh")) + [os.path.join(ROOT, "include", "gccb200.h")]
    objs, procs = [], []
    for src in sources():
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        if force or _stale(obj, [src] + hdrs):
            cmd = [NVCC] + ARCH + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-c", src, "-o", obj]
            procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0 or verbose:
            sys.stderr.write(out.decode())
        failed |= p.returncode != 0
    if failed:
        raise RuntimeError("nvcc failed")
    if force or procs or _stale(LIB, objs):
        subprocess.check_call([NVCC] + ARCH + ["-shared", "-o", LIB] + objs)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
