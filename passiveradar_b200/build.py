"""Build libprcore.so in-tree with nvcc for sm_90a (cross-compiles without a GPU).

    python -m passiveradar_b200.build [--force]

The .so is git-ignored; it is rebuilt whenever a source, header or flag changes (source_hash).
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
LIB = os.path.join(PKG, "libprcore.so")
SOURCES = [os.path.join(CSRC, "prcore.cu")]
# every header prcore.cu includes: a stale library after editing one of them is the worst kind of bug
HEADERS = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + \
          [os.path.join(ROOT, "include", "prcore.h")]

NVCC_FLAGS = [
    "-O3", "-std=c++17",
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-lineinfo",
    "-Xcompiler", "-fPIC", "-shared",
    "-Xptxas", "-v",
]


def find_nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found; libprcore.so cannot be built (there is no CPU fallback)")


HASH = os.path.join(PKG, "libprcore.hash")


def source_hash() -> str:
    """sha256 over every source, header and the compiler flags: what the library was built from.  File times are
    not used -- the snapshot that carries the built library to the GPU box does not keep them."""
    import hashlib
    h = hashlib.sha256(" ".join(NVCC_FLAGS).encode())
    for f in SOURCES + HEADERS:
        h.update(os.path.basename(f).encode())
        with open(f, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def up_to_date() -> bool:
    if not (os.path.exists(LIB) and os.path.exists(HASH)):
        return False
    with open(HASH) as f:
        return f.read().strip() == source_hash()


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and up_to_date():
        return LIB
    tmp = LIB + f".tmp{os.getpid()}"           # concurrent builders (torchrun ranks) never see a half-written library
    cmd = [find_nvcc()] + NVCC_FLAGS + ["-I", os.path.join(ROOT, "include"), "-I", CSRC,
                                          "-o", tmp] + SOURCES
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode == 0:
        os.replace(tmp, LIB)
    if verbose or res.returncode != 0:
        sys.stderr.write(res.stdout + res.stderr)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed building libprcore.so")
    with open(os.path.join(PKG, "libprcore.ptxas.log"), "w") as f:
        f.write(res.stdout + res.stderr)
    with open(HASH, "w") as f:
        f.write(source_hash() + "\n")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
