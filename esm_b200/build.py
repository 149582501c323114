"""In-tree build of libesmb200.so with nvcc for sm_90a (H100) (no JIT cache: the .so travels with the repo snapshot).

    python -m esm_b200.build [--force]
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libesmb200.so")
SOURCES = ["api.cu"]
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [os.path.join("..", "..", "include", "esmb200.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",
    "-O3", "-lineinfo", "-std=c++17",
    "-shared", "-Xcompiler", "-fPIC",
]


def _stale() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS]
    return any(os.path.getmtime(d) > t for d in deps if os.path.exists(d))


def build(force: bool = False, verbose: bool = False, defines=(), out: str = OUT) -> str:
    """Build libesmb200.so.  `defines` / `out` produce developer variants that are loaded through ESMB200_LIB_PATH;
    the product library takes neither."""
    if not force and out == OUT and not _stale():
        return OUT
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        raise RuntimeError("nvcc not found: libesmb200.so must be built with a CUDA 12 toolkit (sm_90a)")
    cmd = ([nvcc] + NVCC_FLAGS + [f"-D{d}" for d in defines] + (["-Xptxas", "-v"] if verbose else []) +
           ["-o", out] + SOURCES)
    r = subprocess.run(cmd, cwd=CSRC, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return out


if __name__ == "__main__":
    defs = [a[2:] for a in sys.argv[1:] if a.startswith("-D")]
    outs = [a.split("=", 1)[1] for a in sys.argv[1:] if a.startswith("--out=")]
    print(build(force="--force" in sys.argv or bool(defs), verbose="-v" in sys.argv, defines=defs,
                out=os.path.abspath(outs[0]) if outs else OUT))
