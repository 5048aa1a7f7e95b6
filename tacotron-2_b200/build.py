"""Builds libt2b200.so (hand-written sm_90a CUDA + the C-ABI) in-tree with nvcc.

The library is plain CUDA C++ with an ``extern "C"`` surface (include/t2b200.h); it links only against the
CUDA runtime, so it cross-compiles on a machine without a GPU.
"""
import hashlib
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
BUILD = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libt2b200.so")
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr",
          "-Xptxas", "-v"] + ARCH


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _digest(path):
    h = hashlib.sha1()
    for f in sorted(os.listdir(CSRC)) + ["../../include/t2b200.h"]:
        p = os.path.join(CSRC, f)
        if os.path.isfile(p):
            h.update(open(p, "rb").read())
    h.update(" ".join(CFLAGS).encode())
    h.update(path.encode())
    return h.hexdigest()


def _compile(src):
    obj = os.path.join(BUILD, src.replace(".cu", ".o"))
    stamp = obj + ".sha1"
    dig = _digest(src)
    if os.path.exists(obj) and os.path.exists(stamp) and open(stamp).read() == dig:
        return obj, ""
    cmd = [NVCC, "-c", os.path.join(CSRC, src), "-o", obj] + CFLAGS
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed for %s:\n%s\n%s" % (src, r.stdout, r.stderr))
    open(stamp, "w").write(dig)
    return obj, r.stderr


def build(verbose=False, force=False):
    os.makedirs(BUILD, exist_ok=True)
    if force:
        for f in os.listdir(BUILD):
            os.remove(os.path.join(BUILD, f))
    srcs = _sources()
    with ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        results = list(ex.map(_compile, srcs))
    objs = [o for o, _ in results]
    log = "\n".join(l for _, l in results if l)
    if verbose and log:
        print(log)
    if log:
        open(os.path.join(BUILD, "ptxas.log"), "a").write(log + "\n")
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-o", LIB] + objs + ARCH + ["-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError("link failed:\n%s\n%s" % (r.stdout, r.stderr))
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
