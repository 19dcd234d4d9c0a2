"""Build libmagma_b200.so (hand-written sm_90a CUDA + the C ABI) in-tree with nvcc.

`python -m magma_b200.build` or `magma_b200.build.build()`. nvcc cross-compiles without a GPU, so this
is also the CPU-side "does it build" check run by `__graft_entry__.build()`. The built library lands in
`magma_b200/lib/` (git-ignored build products).
"""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
OBJDIR = os.path.join(HERE, "lib", "obj")
LIB = os.path.join(LIBDIR, "libmagma_b200.so")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
CFLAGS = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "--expt-relaxed-constexpr"]


def _sources():
    return sorted(f for f in os.listdir(CSRC) if f.endswith(".cu"))


def _headers_mtime():
    m = 0.0
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for f in os.listdir(root):
            if f.endswith((".cuh", ".h", ".hpp")):
                m = max(m, os.path.getmtime(os.path.join(root, f)))
    return m


def _compile_one(src, verbose):
    obj = os.path.join(OBJDIR, src[:-3] + ".o")
    cmd = [NVCC, *ARCH, *CFLAGS, "-c", os.path.join(CSRC, src), "-o", obj]
    if verbose:
        cmd.insert(1, "-Xptxas=-v")
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"nvcc failed for {src}:\n{r.stdout}\n{r.stderr}")
    return obj, r.stderr


def build(force=False, verbose=False):
    """Compile every .cu under csrc/ for sm_90a and link libmagma_b200.so. Returns the library path."""
    os.makedirs(OBJDIR, exist_ok=True)
    srcs = _sources()
    hdr_m = _headers_mtime()
    todo = []
    for s in srcs:
        obj = os.path.join(OBJDIR, s[:-3] + ".o")
        src_m = max(os.path.getmtime(os.path.join(CSRC, s)), hdr_m)
        if force or not os.path.exists(obj) or os.path.getmtime(obj) < src_m:
            todo.append(s)
    logs = []
    if todo:
        with ThreadPoolExecutor(max_workers=min(8, len(todo))) as ex:
            for obj, log in ex.map(lambda s: _compile_one(s, verbose), todo):
                logs.append(log)
    objs = [os.path.join(OBJDIR, s[:-3] + ".o") for s in srcs]
    if todo or not os.path.exists(LIB):
        cmd = [NVCC, *ARCH, "-shared", "-o", LIB, *objs, "-lcudart"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    if verbose:
        print("\n".join(logs))
    return LIB


if __name__ == "__main__":
    p = build(force="--force" in sys.argv, verbose="-v" in sys.argv)
    print(p)
