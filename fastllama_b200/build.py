"""In-tree build of the native libraries (nvcc cross-compiles sm_90a without a GPU)."""
from __future__ import annotations

import os
import subprocess

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
LIB_DIR = os.path.join(PKG, "lib")       # the only place the package loads native code from (tests pass explicit paths to stand-ins)
CSRC = os.path.join(PKG, "csrc")


def lib_path(name: str) -> str:
    return os.path.join(LIB_DIR, name)


def build_all(verbose: bool = False, targets=("all",)) -> None:
    """Compile every native target with make (incremental).  Raises on failure."""
    cmd = ["make", "-C", CSRC, "-j8", *targets]
    res = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if verbose or res.returncode != 0:
        print(res.stdout)
    if res.returncode != 0:
        raise RuntimeError(f"native build failed: {' '.join(cmd)}")
