"""Build the C-ABI shared library (include/sige_b200.h) for sm_90a (H100), in-tree.

    python -m sige_b200.build [--force] [--verbose]

Produces sige_b200/lib/libsige_b200.so with plain `nvcc` (no torch, no cmake): the
library has no dependency on libtorch — PyTorch only supplies device memory and
streams on the Python side.  Replaces reference setup.py:147-182 (which has no arch
flags at all); this build targets exactly one architecture, sm_90a.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB_DIR = os.path.join(HERE, "lib")
LIB_PATH = os.path.join(LIB_DIR, "libsige_b200.so")
OBJ_DIR = os.path.join(HERE, "lib", "_obj")
STAMP = os.path.join(LIB_DIR, "build.stamp")

ARCH = "sm_90a"
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-std=c++17", "-lineinfo",
    "--expt-relaxed-constexpr",
    "-Xcompiler", "-fPIC",
    "-DSIGE_BUILT_ARCH=\"%s\"" % ARCH,
]


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    files = sources() + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith(".cuh")]
    files.append(os.path.join(HERE, "..", "include", "sige_b200.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def up_to_date() -> bool:
    if not (os.path.isfile(LIB_PATH) and os.path.isfile(STAMP)):
        return False
    try:
        return open(STAMP).read().strip() == _digest()
    except OSError:
        return False


def build(force: bool = False, verbose: bool = False) -> str:
    if up_to_date() and not force:
        return LIB_PATH
    if not os.path.isfile(NVCC):
        raise RuntimeError("nvcc not found at %s; cannot build libsige_b200.so" % NVCC)
    os.makedirs(OBJ_DIR, exist_ok=True)
    extra = ["-Xptxas", "-v"] if verbose else []

    def compile_one(src: str) -> str:
        obj = os.path.join(OBJ_DIR, os.path.basename(src)[:-3] + ".o")
        cmd = [NVCC, *NVCC_FLAGS, *extra, "-c", src, "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
        if verbose:
            sys.stderr.write(r.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    cmd = [NVCC, "-shared", "-o", LIB_PATH, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart_static", "-ldl", "-lrt", "-lpthread"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    with open(STAMP, "w") as fh:
        fh.write(_digest())
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="--verbose" in sys.argv))
