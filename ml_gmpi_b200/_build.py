"""In-tree build of the CUDA library (nvcc, sm_90a only).  The .so is git-ignored: build() makes it.

One nvcc call compiles and links the library's three translation units: mpi_render.cu, and the empty-space skipping (mpi_skip.cu)
and uint8-MPI (mpi_u8.cu) kernels it launches.  Without -rdc each file's device code is compiled on its own, so the kernels of one
file keep their machine code whatever the others add."""
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libgmpi_mpi_render.so")
SOURCES = ["mpi_render.cu", "mpi_skip.cu", "mpi_u8.cu"]
HEADERS = ["mpi_common.cuh", "mpi_fwd_staged.cuh", "mpi_fwd_direct.cuh", "mpi_kernel_keys.cuh", "mpi_bwd_box.cuh", "mpi_bwd_direct.cuh",
           "mpi_range_check.cuh", "mpi_light.cuh", "mpi_debug.cuh", "tma_utils.cuh", os.path.join("..", "..", "include", "gmpi_mpi_render.h")]
NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-diag-suppress", "1886", "-shared",
              "-Xcompiler", "-fPIC"]


def nvcc_path():
    p = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(p):
        raise RuntimeError("nvcc not found; cannot build the sm_90a library")
    return p


def is_stale(path: str = LIB_PATH) -> bool:
    if not os.path.exists(path):
        return True
    t = os.path.getmtime(path)
    deps = [os.path.join(CSRC, s) for s in SOURCES + HEADERS] + [os.path.join(CSRC, f) for f in os.listdir(CSRC)]
    return any(os.path.getmtime(d) > t for d in deps if os.path.isfile(d))


def _nvcc(args, verbose):
    res = subprocess.run([nvcc_path()] + args + (["-Xptxas", "-v"] if verbose else []), cwd=CSRC, capture_output=True, text=True)
    if res.returncode != 0:
        raise RuntimeError("nvcc failed:\n" + res.stdout + res.stderr)
    if verbose:
        print(res.stdout + res.stderr)


def build_library(force: bool = False, verbose: bool = False) -> str:
    """Builds the library; returns its path."""
    if force or is_stale(LIB_PATH):
        _nvcc(NVCC_FLAGS + ["-o", LIB_PATH] + SOURCES, verbose)
    return LIB_PATH
