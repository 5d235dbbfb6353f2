"""Build lib3dhg_sm90a.so in-tree with nvcc (sm_90a only; no JIT cache, no fallback)."""
from __future__ import annotations

import glob
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "lib3dhg_sm90a.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def sources():
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")))


def needs_build():
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    deps = sources() + glob.glob(os.path.join(CSRC, "*.cuh")) + [os.path.abspath(__file__)]
    return any(os.path.getmtime(p) > t for p in deps)


def build(force=False, verbose=False):
    if not force and not needs_build():
        return LIB
    objs = []
    procs = []
    os.makedirs(os.path.join(HERE, "build"), exist_ok=True)
    for src in sources():
        obj = os.path.join(HERE, "build", os.path.basename(src)[:-3] + ".o")
        objs.append(obj)
        log = open(obj + ".log", "w")
        procs.append((src, log, subprocess.Popen([NVCC, *FLAGS, "-c", src, "-o", obj], stdout=log, stderr=subprocess.STDOUT)))
    failed = False
    for src, log, p in procs:
        rc = p.wait()
        log.close()
        if rc != 0 or verbose:
            sys.stderr.write(open(log.name).read())
        failed |= rc != 0
    if failed:
        raise RuntimeError("nvcc failed (see messages above)")
    subprocess.check_call([NVCC, "-shared", *FLAGS[:2], "-o", LIB, *objs, "-lcudart"])
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
