"""Builds libpipegcn_b200.so in-tree with nvcc for sm_90a (no torch, no JIT cache).

`python -m pipegcn_b200.build` or `__graft_entry__.build()`.  The shared object, its objects and the stamp of the
sources it was built from are git-ignored: a fresh checkout builds them.
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys
from pathlib import Path

HERE = Path(__file__).resolve().parent
CSRC = HERE / "csrc"
LIB = HERE / "libpipegcn_b200.so"
STAMP = HERE / ".libpipegcn_b200.stamp"

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMPILE_FLAGS = ARCH + ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC"]
LINK_FLAGS = ["--shared", "-cudart", "static"]


def sources():
    return sorted(CSRC.glob("*.cu"))


def _digest() -> str:
    h = hashlib.sha256()
    for p in sorted(list(CSRC.glob("*.cu")) + list(CSRC.glob("*.cuh")) + [HERE.parent / "include" / "pipegcn_b200.h"]):
        h.update(p.name.encode())
        h.update(p.read_bytes())
    h.update(" ".join(COMPILE_FLAGS + LINK_FLAGS).encode())
    return h.hexdigest()


def build(force: bool = False, verbose: bool = True) -> Path:
    dig = _digest()
    if not force and LIB.exists() and STAMP.exists() and STAMP.read_text().strip() == dig:
        return LIB
    nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
    objs = []
    procs = []
    build_dir = HERE / "build"
    build_dir.mkdir(exist_ok=True)
    for src in sources():
        obj = build_dir / (src.stem + ".o")
        cmd = [nvcc] + COMPILE_FLAGS + ["-c", str(src), "-o", str(obj)]
        if verbose:
            print(" ".join(cmd), flush=True)
        procs.append((src, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
        objs.append(str(obj))
    failed = False
    for src, p in procs:
        out, _ = p.communicate()
        if out.strip() and verbose:
            print(out)
        if p.returncode != 0:
            print(out, file=sys.stderr)
            failed = True
    if failed:
        raise RuntimeError("nvcc failed")
    link = [nvcc] + LINK_FLAGS + ["-o", str(LIB)] + objs
    if verbose:
        print(" ".join(link), flush=True)
    subprocess.run(link, check=True)
    STAMP.write_text(dig)
    return LIB


if __name__ == "__main__":
    build(force="--force" in sys.argv)
    print(LIB)
