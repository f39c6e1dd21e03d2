#!/usr/bin/env python
"""Developer tool: build a differently-tuned libgccb200 (extra -D flags) into build_variants/ for
A/B runs on the GPU:  GCCB200_LIB=build_variants/libgccb200_NAME.so python bench.py ..."""
import glob
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from gcc_b200.csrc import build as B  # noqa: E402

name, defs = sys.argv[1], sys.argv[2:]
out_dir = os.path.join(ROOT, "build_variants")
obj_dir = os.path.join(out_dir, "obj_" + name)
os.makedirs(obj_dir, exist_ok=True)
procs, objs = [], []
for src in B.sources():
    obj = os.path.join(obj_dir, os.path.basename(src)[:-3] + ".o")
    objs.append(obj)
    procs.append(subprocess.Popen([B.NVCC] + B.ARCH + B.FLAGS + defs + ["-c", src, "-o", obj]))
assert all(p.wait() == 0 for p in procs)
lib = os.path.join(out_dir, "libgccb200_%s.so" % name)
subprocess.check_call([B.NVCC] + B.ARCH + ["-shared", "-o", lib] + objs)
print(lib)
