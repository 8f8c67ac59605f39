"""Build the CUDA library in-tree with nvcc for sm_90a (H100)."""
from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libcontrolar_b200.so")
SOURCES = ["car_api.cu", "car_vision.cu", "car_train.cu", "gemm.cu"]
# --no-undefined: a kernel launched from one translation unit and defined in another (misc.h) must resolve when the library links
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-shared",
              "-Xcompiler", "-fPIC", "-cudart", "static", "-Xlinker", "--no-undefined"]


def _source_hash(flags) -> str:
    """Content hash of every source the library is built from (+ flags): mtimes do not survive a copy of the tree."""
    import hashlib
    h = hashlib.sha256(" ".join(flags).encode())
    for root in (CSRC, os.path.join(os.path.dirname(HERE), "include")):
        for f in sorted(os.listdir(root)):
            if f.endswith((".cu", ".cuh", ".h")):
                h.update(f.encode())
                with open(os.path.join(root, f), "rb") as fh:
                    h.update(fh.read())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    flags = list(NVCC_FLAGS)
    if os.environ.get("CAR_PK_TRACE"):        # dev: per-phase globaltimer stamps in the persistent decode kernel (CAR_DBG=<step>)
        flags.append("-DPK_TRACE")
    want = _source_hash(flags)
    stamp = LIB + ".srchash"
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == want:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    cmd = [nvcc] + flags + ["-o", LIB] + [os.path.join(CSRC, s) for s in SOURCES]
    if verbose:
        print(" ".join(cmd), flush=True)
    subprocess.run(cmd, check=True)
    with open(stamp, "w") as fh:
        fh.write(want + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
