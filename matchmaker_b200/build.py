"""Build ``libmatchmaker_b200.so`` (hand-written CUDA for sm_90a + the C ABI) in-tree.

    python -m matchmaker_b200.build [--force] [--verbose]

nvcc cross-compiles without a GPU.  The library links the static CUDA runtime only (the
driver entry point for TMA descriptors is resolved at run time), so it loads on a CPU-only
box; every compute entry point then fails loudly with a CUDA error.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
INCLUDE = os.path.join(os.path.dirname(HERE), "include")
LIB_NAME = "libmatchmaker_b200.so"
LIB_PATH = os.path.join(CSRC, LIB_NAME)
OBJ_DIR = os.path.join(CSRC, "build")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC",
    "-Xcompiler", "-fvisibility=hidden",
    "--expt-relaxed-constexpr",
    "-I", INCLUDE,
]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=...)")


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths) -> str:
    h = hashlib.sha256()
    for p in sorted(paths):
        h.update(p.encode())
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def _all_inputs():
    hdrs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hdrs += [os.path.join(INCLUDE, f) for f in os.listdir(INCLUDE) if f.endswith(".h")]
    return sources() + hdrs


def build(force: bool = False, verbose: bool = False, prof: bool = False) -> str:
    """prof=True adds -DMMB200_ENABLE_PROF: the MMB200_*_PROF debugging switches (they allocate and synchronise inside
    the launch path) exist only in such a build, never in the product library."""
    stamp = os.path.join(OBJ_DIR, "stamp.sha256")
    digest = _digest(_all_inputs()) + ("+prof" if prof else "")
    if not force and os.path.isfile(LIB_PATH) and os.path.isfile(stamp) and open(stamp).read() == digest:
        return LIB_PATH
    os.makedirs(OBJ_DIR, exist_ok=True)
    nvcc = _nvcc()
    extra = (["-Xptxas", "-v"] if verbose else []) + (["-DMMB200_ENABLE_PROF"] if prof else [])

    def compile_one(src):
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc, *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    link = [nvcc, "-shared", "-gencode", "arch=compute_90a,code=sm_90a", "-cudart", "static",
            "-Xcompiler", "-fPIC", "-o", LIB_PATH, *objs]
    r = subprocess.run(link, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(digest)
    return LIB_PATH


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    ap.add_argument("--prof", action="store_true", help="debugging build with the MMB200_*_PROF switches compiled in")
    a = ap.parse_args()
    print(build(force=a.force, verbose=a.verbose, prof=a.prof))
