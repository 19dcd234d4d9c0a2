"""TEST INFRASTRUCTURE — builds oracle/_build/libsched_emul.so: the product's host-only schedule files
(magma_b200/csrc/vit_sched.cu and gptj_sched.cu — no kernels, no CUDA calls, see magma_b200/csrc/sched_rt.h), compiled as
plain C++ and linked against oracle/cabi_emul.cpp, the CPU emulation of the primitive C-ABI operators.
tests/test_sched_emul_cpu.py loads it to dry-run the schedules against the oracle. Nothing in magma_b200/ uses it."""
import os
import subprocess

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT_DIR = os.path.join(ROOT, "oracle", "_build")
OUT = os.path.join(OUT_DIR, "libsched_emul.so")
SCHEDULES = [os.path.join(ROOT, "magma_b200", "csrc", "vit_sched.cu"),
             os.path.join(ROOT, "magma_b200", "csrc", "gptj_sched.cu")]
EMUL = os.path.join(ROOT, "oracle", "cabi_emul.cpp")
CUDA_INC = os.environ.get("CUDA_HOME", "/usr/local/cuda") + "/include"   # headers only (types, cudaStream_t)
DEPS = SCHEDULES + [EMUL, os.path.join(ROOT, "magma_b200", "csrc", "sched_rt.h"),
                    os.path.join(ROOT, "include", "magma_b200.h")]


def build(force=False):
    os.makedirs(OUT_DIR, exist_ok=True)
    if not force and os.path.exists(OUT) and os.path.getmtime(OUT) >= max(os.path.getmtime(d) for d in DEPS):
        return OUT
    objs = []
    common = ["g++", "-O2", "-std=c++17", "-fPIC", "-Wall", "-Wno-unknown-pragmas", "-I", CUDA_INC, "-c"]
    jobs = [(src, []) for src in SCHEDULES + [EMUL]]
    for src, extra in jobs:
        obj = os.path.join(OUT_DIR, os.path.basename(src).rsplit(".", 1)[0] + ".o")
        r = subprocess.run(common + extra + ["-x", "c++", src, "-o", obj], capture_output=True, text=True)
        if r.returncode != 0:
            raise RuntimeError(f"g++ failed for {src}:\n{r.stdout}\n{r.stderr}")
        objs.append(obj)
    r = subprocess.run(["g++", "-shared", "-o", OUT, *objs], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout}\n{r.stderr}")
    return OUT


KX_OUT = os.path.join(OUT_DIR, "libkernel_host_exec.so")
KX_SRC = os.path.join(ROOT, "oracle", "kernel_host_exec.cpp")
KX_DEPS = [KX_SRC, os.path.join(ROOT, "include", "magma_b200.h")] + [os.path.join(ROOT, "magma_b200", "csrc", f) for f in ("warp_helpers.cuh", "elt_helpers.cuh",
                                                                          "elt_kernels.cuh", "train_kernels.cuh",
                                                                          "samp_kernels.cuh", "elt_abi.cuh")]


def build_kernel_exec(force=False):
    """oracle/_build/libkernel_host_exec.so: the product's kernel SOURCE (the csrc/*.cuh fragments elementwise.cu includes,
    C-ABI wrappers in elt_abi.cuh included) compiled as host C++ and executed with the CUDA thread model emulated
    (oracle/kernel_host_exec.cpp)."""
    os.makedirs(OUT_DIR, exist_ok=True)
    if not force and os.path.exists(KX_OUT) and os.path.getmtime(KX_OUT) >= max(os.path.getmtime(d) for d in KX_DEPS):
        return KX_OUT
    cmd = ["g++", "-O1", "-std=c++17", "-shared", "-fPIC", "-pthread", "-Wno-unknown-pragmas", "-I", CUDA_INC, "-o", KX_OUT,
           KX_SRC]
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError(f"g++ failed for {KX_SRC}:\n{r.stdout}\n{r.stderr}")
    return KX_OUT


if __name__ == "__main__":
    print(build(force=True))
    print(build_kernel_exec(force=True))
