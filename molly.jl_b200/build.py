"""Build libmollyb200.so in-tree with nvcc for sm_90a (H100, the only target)."""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIB = os.path.join(HERE, "libmollyb200.so")
SOURCES = ["engine.cu"]
# every header under csrc/ plus the C ABI header: an edit to any of them makes the library stale
HEADERS = sorted(f for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))) + [os.path.join("..", "..", "include", "mollyb200.h")]


def _nvcc() -> str:
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found: libmollyb200 cannot be built (there is no CPU fallback)")


def needs_build() -> bool:
    if not os.path.exists(LIB):
        return True
    t = os.path.getmtime(LIB)
    for f in SOURCES + HEADERS:
        if os.path.getmtime(os.path.join(CSRC, f)) > t:
            return True
    return False


def build(force: bool = False, verbose: bool = False, out: str = None) -> str:
    """out: build under another file name next to the default library (e.g. to A/B two versions via MOLLYB200_LIB)."""
    if out is None and not force and not needs_build():
        return LIB
    host_cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    cmd = [
        _nvcc(), "-std=c++17", "-O3", "-lineinfo",
        "-gencode", "arch=compute_90a,code=sm_90a",
        "-ccbin", host_cxx,
        "-Xcompiler", "-fPIC,-O2,-Wall,-Wno-unused-function",
        "--expt-relaxed-constexpr",
        "-shared", "-o", os.path.join(HERE, out) if out else LIB,
    ]
    if verbose:
        cmd += ["-Xptxas", "-v"]
    cmd += [os.path.join(CSRC, s) for s in SOURCES]
    cmd += ["-lcudart"]
    print("[mollyb200] " + " ".join(cmd), file=sys.stderr)
    subprocess.run(cmd, check=True)
    return os.path.join(HERE, out) if out else LIB


if __name__ == "__main__":
    outs = [a[6:] for a in sys.argv[1:] if a.startswith("--out=")]
    build(force="--force" in sys.argv, verbose="-v" in sys.argv, out=outs[0] if outs else None)
