"""In-tree build of libfiber_b200.so (hand-written CUDA for sm_90a, the H100 + the C ABI).

    python -m fiber_b200.build            # or: __graft_entry__.build()

nvcc cross-compiles without a GPU.  The .so lands in fiber_b200/_lib/ (git-ignored build product).
"""
import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "_lib")
SO = os.path.join(LIBDIR, "libfiber_b200.so")
SOURCES = ["engine.cu", "queues.cu", "express.cu", "comm.cu"]
HEADERS = ["kernels.cuh", "bodies.cuh", os.path.join("..", "..", "include", "fiber_b200.h"),
           os.path.join("..", "..", "include", "fiber_b200_body.cuh")]

# every device object of the project (library, body modules, microbenchmarks) is built for this one target:
# the kernels use sm_90a's bulk async copies and mbarriers, and the library refuses any other device
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a"]

NVCC_FLAGS = ARCH_FLAGS + [
    "-O3", "-std=c++17", "-lineinfo",
    "-Xcompiler", "-fPIC,-Wall,-Wno-unused-function",
    "-shared",
    "-I" + CSRC,            # engine.cu includes fiber_b200_body.cuh, which includes kernels.cuh
]
LINK_FLAGS = ["-ldl"]   # body modules (fbr_register_body) and NCCL (fbr_comm_*) are bound at run time


def nvcc():
    for cand in (os.environ.get("NVCC"), shutil.which("nvcc"), "/usr/local/cuda/bin/nvcc"):
        if cand and os.path.exists(cand):
            return cand
    raise RuntimeError("nvcc not found")


def stale():
    if not os.path.exists(SO):
        return True
    t = os.path.getmtime(SO)
    deps = [os.path.join(CSRC, f) for f in SOURCES + HEADERS] + [os.path.abspath(__file__)]
    return any(os.path.getmtime(os.path.normpath(d)) > t for d in deps)


def build(force=False, verbose=False):
    if not force and not stale():
        return SO
    os.makedirs(LIBDIR, exist_ok=True)
    cmd = [nvcc()] + NVCC_FLAGS + (["-Xptxas", "-v"] if verbose else []) + \
        [os.path.join(CSRC, s) for s in SOURCES] + ["-o", SO] + LINK_FLAGS
    subprocess.check_call(cmd)
    return SO


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
