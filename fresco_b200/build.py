"""Build libfresco_b200.so (hand-written sm_90a kernels + C ABI) in-tree with nvcc.

    python -m fresco_b200.build [--force]

nvcc cross-compiles without a GPU; the resulting .so and objects are git-ignored build products.
"""
from __future__ import annotations

import concurrent.futures as cf
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
TAG = os.environ.get("FRESCO_BUILD_TAG", "")                 # A/B builds only: libfresco_b200<TAG>.so next to the product
OBJ = os.path.join(HERE, "csrc", "_obj" + TAG)
LIB = os.path.join(HERE, "libfresco_b200%s.so" % TAG)
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
FLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--use_fast_math=false",
         "-Xptxas", "-v", "-I", os.path.join(os.path.dirname(HERE), "include")]
FLAGS = [f for f in FLAGS if f != "--use_fast_math=false"]
FLAGS += os.environ.get("FRESCO_NVCC_EXTRA", "").split()      # extra nvcc flags for experimental builds


def sources():
    return sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _compile(src, force, verbose):
    obj = os.path.join(OBJ, os.path.basename(src)[:-3] + ".o")
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    headers.append(os.path.join(os.path.dirname(HERE), "include", "fresco_b200.h"))
    if not force and not _stale(obj, [src] + headers):
        return obj, ""
    cmd = [NVCC] + ARCH + FLAGS + ["-c", src, "-o", obj]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    return obj, r.stderr


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    srcs = sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(lambda s: _compile(s, force, verbose), srcs))
    objs = [o for o, _ in results]
    if verbose:
        for _, log in results:
            if log:
                sys.stderr.write(log)
    if force or _stale(LIB, objs):
        cmd = [NVCC] + ARCH + ["-shared", "-o", LIB] + objs + ["-lcudart_static", "-lpthread", "-ldl", "-lrt"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
