"""Builds libjorldy_b200.so (the C-ABI CUDA library) in-tree with nvcc for sm_90a (H100).

No torch involvement: the library is plain CUDA runtime + extern "C" entry points declared in
include/jorldy_b200.h.  Objects are cached under jorldy_b200/lib/obj and rebuilt when a source
(or any header) is newer than the object.
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(LIBDIR, "obj")
LIB = os.path.join(LIBDIR, "libjorldy_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-lineinfo", "-std=c++17", "-Xcompiler", "-fPIC,-fvisibility=hidden", "--expt-relaxed-constexpr"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    hs = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".cuh", ".h"))]
    hs.append(os.path.join(os.path.dirname(HERE), "include", "jorldy_b200.h"))
    return max((os.path.getmtime(h) for h in hs if os.path.exists(h)), default=0.0)


def _compile(src, verbose):
    obj = os.path.join(OBJDIR, src[:-3] + ".o")
    cmd = [NVCC, *ARCH, *CFLAGS, "-I", os.path.join(os.path.dirname(HERE), "include"), "-c",
           os.path.join(CSRC, src), "-o", obj]
    if verbose:
        print(" ".join(cmd), flush=True)
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj


def build(force=False, verbose=False):
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = _sources()
    hm = _headers_mtime()
    todo = []
    for s in srcs:
        obj = os.path.join(OBJDIR, s[:-3] + ".o")
        sm = max(os.path.getmtime(os.path.join(CSRC, s)), hm)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < sm:
            todo.append(s)
    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            list(ex.map(lambda s: _compile(s, verbose), todo))
    objs = [os.path.join(OBJDIR, s[:-3] + ".o") for s in srcs]
    if todo or not os.path.exists(LIB) or any(os.path.getmtime(o) > os.path.getmtime(LIB) for o in objs):
        cmd = [NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-cudart", "static"]
        if verbose:
            print(" ".join(cmd), flush=True)
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
