"""In-tree build of the C-ABI shared library (nvcc, sm_90a only).

`python -m hero_b200.build` compiles every `csrc/*.cu` into `hero_b200/libhero_b200.so`.
nvcc cross-compiles without a GPU, so this also runs on a machine without one; the resulting
`.so` and the object files under `hero_b200/build/` are git-ignored.
"""
import hashlib
import os
import shutil
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
BUILD_DIR = os.path.join(PKG_DIR, "build")
LIB_PATH = os.path.join(PKG_DIR, "libhero_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo", "-O3", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc():
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found; cannot build libhero_b200.so")
    return nvcc


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(paths):
    h = hashlib.sha256()
    for p in paths:
        with open(p, "rb") as f:
            h.update(f.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def build(force=False, verbose=False):
    """Compile changed translation units and link the shared library. Returns its path."""
    os.makedirs(BUILD_DIR, exist_ok=True)
    nvcc = _nvcc()
    headers = sorted(
        [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
        + [os.path.join(PKG_DIR, "..", "include", "hero_b200.h")])
    objs, jobs = [], []
    for src in _sources():
        sp = os.path.join(CSRC, src)
        obj = os.path.join(BUILD_DIR, src[:-3] + ".o")
        stamp = obj + ".sha"
        dig = _digest([sp] + headers)
        objs.append(obj)
        old = open(stamp).read() if os.path.exists(stamp) else ""
        if force or old != dig or not os.path.exists(obj):
            jobs.append((sp, obj, stamp, dig))

    def compile_one(job):
        sp, obj, stamp, dig = job
        cmd = [nvcc] + NVCC_FLAGS + ["-c", sp, "-o", obj]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {sp}:\n{r.stdout}\n{r.stderr}")
        with open(stamp, "w") as f:
            f.write(dig)

    if jobs:
        with ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(compile_one, jobs))
    if jobs or not os.path.exists(LIB_PATH):
        cmd = [nvcc, "-shared", "-o", LIB_PATH] + objs
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    path = build(force="--force" in sys.argv, verbose=True)
    print("built", path)
