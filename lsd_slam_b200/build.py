"""Build the sm_90a (H100) shared library (liblsdgpu.so) in-tree with nvcc.  No GPU needed (cross-compiles)."""
from __future__ import annotations

import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
CSRC = os.path.join(HERE, "csrc")
SRCS = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))     # one unit per subsystem
OUT = os.path.join(HERE, "liblsdgpu.so")
DEPS = [os.path.join(CSRC, f) for f in os.listdir(CSRC)] + [os.path.join(ROOT, "include", "lsdgpu.h")]

NVCC_FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17",
    # parity build: no FMA contraction, IEEE div/sqrt (defaults) -> per-pixel results are bit-identical to a
    # strict-IEEE CPU evaluation of the same expression order (DESIGN.md section 5)
    "--fmad=false",
    "-Xcompiler", "-fPIC", "-shared",
]


def nvcc_path() -> str:
    for c in (shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def needs_build() -> bool:
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.getmtime(d) > t for d in DEPS)


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not needs_build():
        return OUT
    cmd = [nvcc_path()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT] + SRCS
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout + r.stderr)
    if verbose:
        print(r.stderr)
    return OUT


HOST_SRC = os.path.join(HERE, "host", "lsd_host.cpp")
HOST_OUT = os.path.join(HERE, "liblsdgpu_host.so")
DEMO_SRC = os.path.join(HERE, "host", "host_demo.cpp")
DEMO_OUT = os.path.join(HERE, "host_demo")


def build_host(force: bool = False) -> str:
    """C++ host classes (reference call signatures) + the demo driver; plain g++, links liblsdgpu.so."""
    srcs = [HOST_SRC, DEMO_SRC, os.path.join(HERE, "host", "lsd_host.h"), OUT]
    if not force and os.path.exists(HOST_OUT) and os.path.exists(DEMO_OUT) and \
            all(os.path.getmtime(x) <= min(os.path.getmtime(HOST_OUT), os.path.getmtime(DEMO_OUT)) for x in srcs):
        return HOST_OUT
    common = ["g++", "-std=c++17", "-O2", "-Wall", "-Wl,-rpath,$ORIGIN", "-L" + HERE]
    for cmd in (common + ["-fPIC", "-shared", "-o", HOST_OUT, HOST_SRC, "-l:liblsdgpu.so"],
                common + ["-o", DEMO_OUT, DEMO_SRC, "-l:liblsdgpu_host.so", "-l:liblsdgpu.so"]):
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("g++ failed:\n" + r.stdout + r.stderr)
    return HOST_OUT


if __name__ == "__main__":
    print(build(force=True, verbose=True))
    print(build_host(force=True))
