"""In-tree nvcc build of liblade_sm100.so (sm_90a only: the H100; the library keeps its historical name).

The shared library is a plain C-ABI (include/lade_sm100.h); no torch headers are involved, so the
build is a single nvcc invocation that also works on a GPU-less box (cross-compile).
"""
from __future__ import annotations

import hashlib
import os
import shutil
import subprocess
import sys

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_DIR = os.path.join(PKG_DIR, "lib")
LIB_PATH = os.path.join(LIB_DIR, "liblade_sm100.so")
STAMP = os.path.join(LIB_DIR, "liblade_sm100.stamp")
SOURCES = ["state.cu", "sampling.cu", "capture.cu","layer_ops.cu", "attn_mma.cu", "attn_tc.cu", "attn_api.cu", "gemm_tc.cu", "lp_nccl.cu"]
NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC", "-ldl",
]


def _find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.isfile(cand):
            return cand
    raise RuntimeError("nvcc not found (set NVCC=...)")


def _source_hash() -> str:
    h = hashlib.sha256()
    files = [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cu", ".cuh", ".h"))]
    files.append(os.path.join(os.path.dirname(PKG_DIR), "include", "lade_sm100.h"))
    for f in files:
        with open(f, "rb") as fh:
            h.update(os.path.basename(f).encode())     # names, not absolute paths: the tree is relocatable
            h.update(fh.read())
    h.update(" ".join(NVCC_FLAGS).encode())
    return h.hexdigest()


def is_fresh() -> bool:
    if not (os.path.isfile(LIB_PATH) and os.path.isfile(STAMP)):
        return False
    with open(STAMP) as f:
        return f.read().strip() == _source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    """Compile csrc/*.cu -> lib/liblade_sm100.so if sources changed. Returns the library path."""
    if not force and is_fresh():
        return LIB_PATH
    os.makedirs(LIB_DIR, exist_ok=True)
    # Several ranks may get here at once (torchrun): serialise on a lock file, re-check under the lock, and publish the
    # library with an atomic rename so no process can ever dlopen a half-written file.
    import fcntl
    with open(os.path.join(LIB_DIR, ".build.lock"), "w") as lock:
        fcntl.flock(lock, fcntl.LOCK_EX)
        try:
            if not force and is_fresh():
                return LIB_PATH
            tmp = LIB_PATH + f".tmp.{os.getpid()}"
            cmd = [_find_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
                  ["-o", tmp] + [os.path.join(CSRC, s) for s in SOURCES]
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                if os.path.exists(tmp):
                    os.remove(tmp)
                raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
            if verbose:
                print(res.stderr)
            if os.path.exists(STAMP):
                os.remove(STAMP)
            os.replace(tmp, LIB_PATH)
            with open(STAMP + ".tmp", "w") as f:
                f.write(_source_hash())
            os.replace(STAMP + ".tmp", STAMP)
        finally:
            fcntl.flock(lock, fcntl.LOCK_UN)
    return LIB_PATH


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
