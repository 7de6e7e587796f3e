# -*- coding: utf-8 -*-
"""
In-tree build of ``george_b200/lib/libbgp_b200.so`` with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m george_b200._build [--force] [--verbose]

The shared library is plain C ABI (``include/bgp.h``); it links only the CUDA runtime (static) so it loads in any
process.  Object files are cached per translation unit under ``george_b200/lib/obj`` and rebuilt when a source or
header is newer.
"""

import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIBDIR = os.path.join(_HERE, "lib")
LIB = os.path.join(LIBDIR, "libbgp_b200.so")
INCLUDE = os.path.join(os.path.dirname(_HERE), "include")

SOURCES = ["core.cu", "kmat.cu", "kmat_ops.cu", "dense.cu", "hodlr.cu", "hodlr_sym.cu", "comm.cu", "sample.cu"]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-O3",
    "--expt-relaxed-constexpr",
    "-Xptxas", "-v",
]


def _nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: cannot build libbgp_b200.so (there is no CPU fallback)")


def _newest_header():
    t = 0.0
    for d in (CSRC, INCLUDE):
        for f in os.listdir(d):
            if f.endswith((".cuh", ".h")):
                t = max(t, os.path.getmtime(os.path.join(d, f)))
    return t


def build(force=False, verbose=False):
    nvcc = _nvcc()
    objdir = os.path.join(LIBDIR, "obj")
    os.makedirs(objdir, exist_ok=True)
    hdr_t = _newest_header()
    jobs = []
    objs = []
    for src in SOURCES:
        sp = os.path.join(CSRC, src)
        if not os.path.exists(sp):
            continue
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        objs.append(obj)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < max(os.path.getmtime(sp), hdr_t):
            jobs.append((sp, obj))

    def compile_one(job):
        sp, obj = job
        cmd = [nvcc] + NVCC_FLAGS + ["-I", INCLUDE, "-c", sp, "-o", obj]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
        log = os.path.join(objdir, os.path.basename(sp) + ".ptxas.log")
        with open(log, "w") as fh:  # build artefact (git-ignored): registers / shared memory / spills per kernel
            fh.write("".join(l for l in r.stdout.splitlines(True) if "Compile time" not in l))
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for {0}:\n{1}".format(sp, r.stdout))
        if verbose:
            print(r.stdout)
        return obj

    if jobs:
        with ThreadPoolExecutor(max_workers=min(4, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or not os.path.exists(LIB):
        cmd = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-o", LIB] + objs + ["-ldl"]
        r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, universal_newlines=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n" + r.stdout)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
