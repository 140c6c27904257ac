"""Build libfo1.so (sm_90a) in-tree with nvcc.  No torch extension machinery: the product is a
plain C-ABI shared library loaded through ctypes."""
from __future__ import annotations

import concurrent.futures as cf
import hashlib
import os
import shutil
import subprocess
import sys

PKG = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(PKG)
CSRC = os.path.join(PKG, "csrc")
OBJ = os.path.join(PKG, "build")
LIB = os.path.join(PKG, "libfo1.so")

NVCC = os.environ.get("NVCC") or shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
FLAGS = [
    "-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC", "-Xcompiler", "-Wall", "--expt-relaxed-constexpr",
    "-I", os.path.join(REPO, "include"), "-I", CSRC,
]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _stamp(path: str) -> str:
    h = hashlib.sha1()
    h.update(" ".join(FLAGS).encode())
    deps = [path] + [os.path.join(CSRC, f) for f in sorted(os.listdir(CSRC)) if f.endswith((".cuh", ".h"))]
    deps.append(os.path.join(REPO, "include", "fo1.h"))
    for d in deps:
        with open(d, "rb") as fh:
            h.update(fh.read())
    return h.hexdigest()


def _compile(src: str, verbose: bool) -> str:
    path = os.path.join(CSRC, src)
    obj = os.path.join(OBJ, src[:-3] + ".o")
    stamp_file = obj + ".stamp"
    stamp = _stamp(path)
    if os.path.exists(obj) and os.path.exists(stamp_file) and open(stamp_file).read() == stamp:
        return obj
    cmd = [NVCC, *FLAGS, "-c", path, "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    if verbose or r.stderr.strip():
        sys.stderr.write(r.stderr)
    with open(stamp_file, "w") as fh:
        fh.write(stamp)
    return obj


def build(verbose: bool = False, force: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    if force:
        for f in os.listdir(OBJ):
            os.remove(os.path.join(OBJ, f))
    srcs = _sources()
    with cf.ThreadPoolExecutor(max_workers=min(8, len(srcs))) as ex:
        objs = list(ex.map(lambda s: _compile(s, verbose), srcs))
    newest = max(os.path.getmtime(o) for o in objs)
    if force or not os.path.exists(LIB) or os.path.getmtime(LIB) < newest:
        cmd = [NVCC, "-shared", "-o", LIB, *objs, "-gencode", "arch=compute_90a,code=sm_90a", "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(verbose="-v" in sys.argv, force="-f" in sys.argv))
