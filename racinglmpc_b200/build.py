"""In-tree build of liblmpc_b200.so (nvcc, sm_90a only).  No JIT cache: the .so sits next to this
file, inside the package, so that the package imports from the repository tree."""
import os
import shutil
import subprocess

HERE = os.path.dirname(os.path.abspath(__file__))
SRC = os.path.join(HERE, "csrc", "lmpc_b200.cu")
DEPS = [SRC] + [os.path.join(HERE, "csrc", f) for f in ("ftocp_pdip.cuh", "safeset.cuh", "lapbooks.cuh", "probe.cuh")] + \
       [os.path.join(HERE, "..", "include", "lmpc_b200.h"), os.path.abspath(__file__)]   # this file holds the architecture flags
OUT = os.path.join(HERE, "liblmpc_b200.so")
CUDA_HOME = os.environ.get("CUDA_HOME", "/usr/local/cuda")
NVCC = os.environ.get("NVCC", os.path.join(CUDA_HOME, "bin", "nvcc"))
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]      # H100 (Hopper); the kernels use sm_90 PTX (cp.async.bulk, mbarrier)
FLAGS = ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC", "-shared"]


def stale():
    if not os.path.exists(OUT):
        return True
    t = os.path.getmtime(OUT)
    return any(os.path.exists(d) and os.path.getmtime(d) > t for d in DEPS)


def build_native(force=False, verbose=False):
    if not force and not stale():
        return OUT
    cxx = shutil.which("g++")
    cmd = [NVCC] + FLAGS + (["-ccbin", cxx] if cxx else []) + (["-Xptxas", "-v"] if verbose else []) + ["-o", OUT, SRC]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + r.stdout)
    if verbose:
        print(r.stdout)
    return OUT


if __name__ == "__main__":
    build_native(force=True, verbose=True)
