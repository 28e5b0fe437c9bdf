"""Builds libhi3d_b200.so (the C-ABI CUDA library) in-tree with nvcc for the H100 (sm_90a).

`nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo` per translation unit (parallel), then one
`nvcc -shared` link.  No torch headers are involved: the library is plain CUDA behind `include/hi3d_b200.h`
and is loaded with ctypes (`_native.py`).  The .so, its digest stamp and the object files are build products
(git-ignored).
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
INC = os.path.join(os.path.dirname(HERE), "include")
LIB = os.path.join(HERE, "libhi3d_b200.so")
STAMP = LIB + ".sha256"                 # digest of what LIB was built from
OBJ = os.path.join(HERE, "build")
SOURCES = ["gemm_mma.cu", "gemm_tc5.cu", "attn.cu", "attn_tc5.cu", "attn_fp8_tc5.cu", "norm.cu", "misc.cu", "peer.cu", "attn512_tc5.cu",
           "attn_d80_tc5.cu", "dpt.cu", "u2net.cu"]
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
NVCC_FLAGS = ARCH + ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr", "-I", INC]


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found; cannot build libhi3d_b200.so")


def _digest() -> str:
    """sha256 of every source, the public header and the compiler flags: the build identity of the library.  File times are
    not used, so a built tree that is copied or checked out elsewhere (new times) is still recognised as built."""
    h = hashlib.sha256(" ".join(ARCH + NVCC_FLAGS[len(ARCH):-2]).encode())
    for f in sorted(os.listdir(CSRC)) + ["../../include/hi3d_b200.h"]:
        h.update(f.encode())
        with open(os.path.join(CSRC, f), "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def is_fresh() -> bool:
    try:
        with open(STAMP) as f:
            return os.path.exists(LIB) and f.read().strip() == _digest()
    except OSError:
        return False


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and is_fresh():
        return LIB
    nvcc = _nvcc()
    os.makedirs(OBJ, exist_ok=True)

    def cc(src):
        o = os.path.join(OBJ, src.replace(".cu", ".o"))
        cmd = [nvcc] + NVCC_FLAGS + ["-c", os.path.join(CSRC, src), "-o", o]
        if verbose:
            cmd.insert(1, "-Xptxas=-v")
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
        if verbose:
            sys.stderr.write(r.stderr)
        return o

    with ThreadPoolExecutor(max_workers=min(8, len(SOURCES))) as ex:
        objs = list(ex.map(cc, SOURCES))
    r = subprocess.run([nvcc, "-shared"] + ARCH + ["-o", LIB] + objs,
                       capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    with open(STAMP, "w") as f:
        f.write(_digest() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
