"""In-tree build of libllamagen_b200.so (sm_90a only).

nvcc cross-compiles without a GPU; the resulting .so has no dependency on libcuda/libcudart at load
time (cudart is linked statically, driver entry points are resolved lazily), so it can be dlopen'ed on
a CPU-only box for the ABI tests.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT_DIR = os.path.join(HERE, os.environ.get("LG_LIB_DIR", "lib"))
LIB = os.path.join(OUT_DIR, "libllamagen_b200.so")
EXTRA_DEFS = os.environ.get("LG_NVCC_DEFS", "").split()
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
          "--expt-extended-lambda", "-Xptxas", "-v"]


def sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for f in sorted(os.listdir(CSRC)):
        if f.endswith((".cu", ".cuh", ".h")):
            h.update(f.encode())
            h.update(open(os.path.join(CSRC, f), "rb").read())
    h.update(open(os.path.join(HERE, "..", "include", "llamagen_b200.h"), "rb").read())
    h.update(" ".join(ARCH + CFLAGS + EXTRA_DEFS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OUT_DIR, exist_ok=True)
    stamp = os.path.join(OUT_DIR, "build.sha256")
    dig = _digest()
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        return LIB
    if not os.path.exists(NVCC):
        raise RuntimeError(f"nvcc not found at {NVCC}; cannot build {LIB}")
    objs = []

    def compile_one(src):
        obj = os.path.join(OUT_DIR, src.replace(".cu", ".o"))
        cmd = [NVCC, *ARCH, *CFLAGS, *EXTRA_DEFS, "-c", os.path.join(CSRC, src), "-o", obj]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log = os.path.join(OUT_DIR, src.replace(".cu", ".ptxas.log"))
        with open(log, "w") as f:
            f.write(r.stdout + r.stderr)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            print(f"[build] {src} ok", file=sys.stderr)
        return obj

    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        objs = list(ex.map(compile_one, sources()))
    cmd = [NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-cudart", "static"]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(stamp, "w") as f:
        f.write(dig)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
