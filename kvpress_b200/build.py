"""Builds libkvpress_b200.so (the C-ABI library of include/kvpress_b200.h) in-tree with nvcc.

sm_90a (H100) only: `-gencode arch=compute_90a,code=sm_90a`. No torch headers are involved; the
library is plain CUDA C++ behind an extern "C" surface, loaded from Python with ctypes.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

PKG_DIR = Path(__file__).resolve().parent
CSRC = PKG_DIR / "csrc"
LIB_PATH = PKG_DIR / "libkvpress_b200.so"
STAMP = PKG_DIR / "build" / "stamp.txt"
SOURCES = ["api.cu", "knorm.cu", "knorm_cluster.cu", "keydiff.cu", "select_compact.cu", "snapkv.cu", "expected_attention.cu",
           "criticalkv.cu", "observed_attention.cu", "non_causal_attention.cu", "lagkv.cu", "cur.cu", "merging.cu",
           "think.cu", "finch.cu", "cam.cu", "kvzap.cu", "tmap.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if cand and (os.path.isabs(cand) and os.path.exists(cand) or not os.path.isabs(cand)):
            return cand
    raise RuntimeError("nvcc not found")


def _fingerprint() -> str:
    h = hashlib.sha256()
    files = sorted(CSRC.glob("*.cu")) + sorted(CSRC.glob("*.cuh")) + [
        PKG_DIR.parent / "include" / "kvpress_b200.h", Path(__file__)]
    for f in files:
        h.update(f.name.encode())
        h.update(f.read_bytes())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> Path:
    """Compile every .cu into objects and link the shared library. Incremental by content hash."""
    fp = _fingerprint()
    if not force and LIB_PATH.exists() and STAMP.exists() and STAMP.read_text() == fp:
        return LIB_PATH
    obj_dir = PKG_DIR / "build"
    obj_dir.mkdir(exist_ok=True)
    nvcc = _nvcc()
    procs = []
    objs = []
    for src in SOURCES:
        obj = obj_dir / (src.replace(".cu", ".o"))
        objs.append(str(obj))
        cmd = [nvcc, *NVCC_FLAGS, "-c", str(CSRC / src), "-o", str(obj)]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if out and (verbose or p.returncode != 0):
            sys.stderr.write(out.decode())
        if p.returncode != 0:
            failed = True
            sys.stderr.write(f"nvcc failed on {src}\n")
    if failed:
        raise RuntimeError("kvpress_b200: CUDA build failed")
    link = [nvcc, "-gencode", "arch=compute_90a,code=sm_90a", "-shared", "-cudart", "static", "-o", str(LIB_PATH), *objs]
    subprocess.run(link, check=True)
    STAMP.write_text(fp)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
