"""In-tree build of libpcl_b200.so (sm_90a only) with plain nvcc — no torch headers, no JIT cache.

    python -m contrastiveseg_b200.build [--force]

The built library stays next to the sources (contrastiveseg_b200/lib/) so that it travels with a
repo snapshot; it is git-ignored.  nvcc cross-compiles without a GPU.
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIBNAME = "libpcl_b200.so"
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
              "-Xptxas", "-v"]


def _nvcc() -> str:
    cand = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(cand):
        raise RuntimeError("nvcc not found (set $NVCC)")
    return cand


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                h.update(f.encode())
                h.update(open(os.path.join(root, f), "rb").read())
    h.update(" ".join(ARCH_FLAGS + NVCC_FLAGS).encode())
    return h.hexdigest()


def library_path() -> str:
    return os.path.join(LIBDIR, LIBNAME)


def is_current() -> bool:
    stamp = os.path.join(LIBDIR, "build.sha256")
    return os.path.exists(library_path()) and os.path.exists(stamp) and open(stamp).read().strip() == _digest()


def build_library(force: bool = False, verbose: bool = False) -> str:
    if not force and is_current():
        return library_path()
    os.makedirs(OBJDIR, exist_ok=True)
    nvcc = _nvcc()
    srcs = sources()
    logs = {}

    def compile_one(src):
        obj = os.path.join(OBJDIR, os.path.basename(src)[:-3] + ".o")
        cmd = [nvcc] + ARCH_FLAGS + NVCC_FLAGS + ["-I", os.path.join(HERE, "..", "include"), "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        logs[src] = r.stdout + r.stderr
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        return obj

    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(compile_one, srcs))
    out = library_path()
    cmd = [nvcc] + ARCH_FLAGS + ["-shared", "-o", out] + objs + ["-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(os.path.join(LIBDIR, "ptxas.log"), "w") as f:
        for s in srcs:
            f.write(f"==== {os.path.basename(s)}\n{logs[s]}\n")
    with open(os.path.join(LIBDIR, "build.sha256"), "w") as f:
        f.write(_digest())
    if verbose:
        print(open(os.path.join(LIBDIR, "ptxas.log")).read())
    return out


if __name__ == "__main__":
    p = build_library(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
