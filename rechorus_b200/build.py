"""Build libb200rec.so in-tree with nvcc for sm_90a (H100; cross-compiles without a GPU).

    python -m rechorus_b200.build [--force] [--verbose]

The .so is git-ignored and rebuilt from source by every checkout.  Objects go to build/.
"""
from __future__ import annotations

import argparse
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

PKG = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ_DIR = os.path.join(ROOT, "build", "obj")
LIB_PATH = os.path.join(PKG, "libb200rec.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden",
          "--expt-relaxed-constexpr", "-Xptxas", "-v"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _newest_header_mtime():
    m = 0.0
    for d in (CSRC, os.path.join(ROOT, "include")):
        for f in os.listdir(d):
            if f.endswith((".cuh", ".h")):
                m = max(m, os.path.getmtime(os.path.join(d, f)))
    return m


def _compile(src, force, verbose):
    obj = os.path.join(OBJ_DIR, src[:-3] + ".o")
    spath = os.path.join(CSRC, src)
    if (not force and os.path.exists(obj)
            and os.path.getmtime(obj) >= max(os.path.getmtime(spath), _newest_header_mtime())):
        return obj, False, ""
    cmd = [NVCC, *ARCH, *CFLAGS, "-c", spath, "-o", obj]
    res = subprocess.run(cmd, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{res.stdout}\n{res.stderr}")
    if verbose:
        print(res.stderr)
    with open(os.path.join(OBJ_DIR, src[:-3] + ".ptxas.txt"), "w") as f:
        f.write(res.stderr)
    return obj, True, res.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ_DIR, exist_ok=True)
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    objs = [r[0] for r in results]
    rebuilt = any(r[1] for r in results)
    if rebuilt or not os.path.exists(LIB_PATH) or force:
        cmd = [NVCC, *ARCH, "-shared", "-o", LIB_PATH, *objs, "-Xlinker", "--exclude-libs=ALL"]
        res = subprocess.run(cmd, capture_output=True, text=True)
        if res.returncode != 0:
            raise RuntimeError(f"link failed:\n{res.stdout}\n{res.stderr}")
    return LIB_PATH


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--force", action="store_true")
    ap.add_argument("--verbose", action="store_true")
    a = ap.parse_args()
    print(build(a.force, a.verbose))
