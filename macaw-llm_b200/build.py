"""Build libmacaw_b200.so (sm_90a only) in-tree with nvcc.

The library has no torch dependency: it is plain CUDA behind the C ABI in include/macaw_b200.h, linked against the
static CUDA runtime so that it can be dlopen()ed on a box without a GPU (symbol checks in the CPU test tier).
"""
from __future__ import annotations

import concurrent.futures
import fcntl
import hashlib
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "build")
LIB = os.path.join(HERE, "libmacaw_b200.so")

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-Xcompiler", "-fPIC",
    "--expt-relaxed-constexpr",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libmacaw_b200.so cannot be built")


def source_files():
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))]
    files.append(os.path.join(HERE, "..", "include", "macaw_b200.h"))
    return files


def source_hash() -> str:
    """Content hash of every kernel source + the ABI header (mtimes do not survive a snapshot copy to the GPU box).
    Compiled into the library (mm_build_hash()) so a stale .so is detected at load time."""
    h = hashlib.sha256()
    for f in source_files():
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()[:16]


def _newer(src_files, target) -> bool:
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(s) > t for s in src_files)


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile + link under an exclusive file lock (ranks of one torchrun job may race here on a fresh checkout); the
    library is linked to a temporary name and renamed into place, so a concurrent dlopen never sees a partial file."""
    os.makedirs(BUILD, exist_ok=True)
    with open(os.path.join(BUILD, ".lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            return _build_locked(force, verbose)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)


def built_hash() -> str:
    try:
        with open(LIB + ".hash") as f:
            return f.read().strip()
    except OSError:
        return ""


def _build_locked(force: bool, verbose: bool) -> str:
    want = source_hash()
    if not force and os.path.exists(LIB) and built_hash() == want:
        return LIB  # another rank built it while we waited for the lock, or nothing changed
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(HERE, "..", "include", "macaw_b200.h"))
    sources = sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))
    objs, jobs = [], []
    for s in sources:
        src = os.path.join(CSRC, s)
        obj = os.path.join(BUILD, s[:-3] + ".o")
        objs.append(obj)
        extra = [f'-DMM_SRC_HASH="{want}"'] if s == "api.cu" else []
        if force or s == "api.cu" or _newer([src] + headers, obj):
            jobs.append([nvcc] + NVCC_FLAGS + extra + ["-c", src, "-o", obj])

    def run(cmd):
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("nvcc failed:\n" + " ".join(cmd) + "\n" + r.stdout + r.stderr)
        return r

    if jobs:
        with concurrent.futures.ThreadPoolExecutor(max_workers=min(8, len(jobs))) as ex:
            list(ex.map(run, jobs))
    tmp = LIB + f".tmp{os.getpid()}"
    run([nvcc, "-shared", "-o", tmp] + objs + ["-gencode", "arch=compute_90a,code=sm_90a", "-ldl"])
    os.replace(tmp, LIB)
    with open(LIB + ".hash.tmp", "w") as f:
        f.write(want + "\n")
    os.replace(LIB + ".hash.tmp", LIB + ".hash")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
