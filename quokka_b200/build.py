"""Builds quokka_b200/libqk.so (the C-ABI library, include/qk.h) with nvcc for sm_90a (H100), in-tree.

The .so is a build product and git-ignored.  nvcc cross-compiles without a GPU, so the library can be
built on a machine that has none (`__graft_entry__.build()`).
"""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libqk.so")
SOURCES = ["abi.cu", "offsets.cu", "synth.cu", "scan.cu", "compact.cu", "partition.cu", "exchange.cu", "join.cu", "hashagg.cu", "asof.cu", "window.cu", "topk.cu", "parquet.cu", "gram.cu", "quantile.cu", "knn.cu", "pattern.cu", "sort.cu", "shift.cu"]
GENCODE = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-std=c++17", *GENCODE, "-lineinfo", "-O3",
              # no FMA contraction: projected fp64 columns are bit-identical to the numpy oracle
              "-fmad=false", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.sep not in cand or os.path.exists(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(HERE, "..", "include", "qk.h"), __file__]
    return any(os.path.getmtime(d) > t for d in deps)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    objdir = os.path.join(HERE, "build")
    os.makedirs(objdir, exist_ok=True)
    nvcc = _nvcc()
    procs = []
    for src in SOURCES:
        obj = os.path.join(objdir, src.replace(".cu", ".o"))
        cmd = [nvcc, *NVCC_FLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((src, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    objs = []
    for src, obj, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {src}:\n{out.decode()}")
        objs.append(obj)
    # extern "C" entry points are the only exported symbols (default visibility restored for them below)
    cmd = [nvcc, "-shared", *GENCODE, "-Xcompiler", "-fPIC", "-o", OUT + ".tmp", *objs]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout.decode()}")
    os.replace(OUT + ".tmp", OUT)
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
