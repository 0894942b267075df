"""In-tree build of the native engine: nvcc -> alicevision_b200/libb200match.so (sm_90a only).

The .so is a build product (git-ignored): build() compiles it next to the sources, and a tree built once is used as is.
"""
from __future__ import annotations

import os
import shutil
import subprocess

_HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(_HERE, "csrc")
LIB = os.path.join(_HERE, "libb200match.so")
SOURCES = ["engine.cu", "acransac_f10.cu", "voctree.cu", "io.cpp"]
def _deps():
    """Every file the library is built from: all of csrc/ and the public headers (a forgotten header here once shipped a stale .so)."""
    import glob
    return sorted(glob.glob(os.path.join(CSRC, "*.cu")) + glob.glob(os.path.join(CSRC, "*.cuh")) + glob.glob(os.path.join(CSRC, "*.cpp"))
                  + glob.glob(os.path.join(CSRC, "*.h")) + glob.glob(os.path.join(_HERE, "..", "include", "*.h")) + [os.path.abspath(__file__)])

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a",   # explicit form: `-arch=sm_90a` also emits compute_90 PTX, which rejects wgmma
    "-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared",
]


def _nvcc() -> str:
    for cand in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def stale() -> bool:
    if not os.path.exists(LIB):
        return True
    if os.environ.get("B200M_NO_BUILD"):       # use the library as built, whatever the source timestamps say (e.g. a read-only tree)
        return False
    t = os.path.getmtime(LIB)
    return any(os.path.getmtime(f) > t for f in _deps())


def build_native(force: bool = False, verbose: bool = False) -> str:
    """Compile the CUDA engine if sources are newer than the library. Returns the library path."""
    if not force and not stale():
        return LIB
    env = dict(os.environ)
    env.pop("CXX", None); env.pop("CC", None)       # nvcc picks its host compiler itself; a CXX wrapper without OpenMP specs breaks it
    cmd = [_nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + [os.path.join(CSRC, s) for s in SOURCES] + ["-o", LIB]
    r = subprocess.run(cmd, env=env, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return LIB


if __name__ == "__main__":
    print(build_native(force=True, verbose=True))
