"""In-tree build of the CUDA library (nvcc, sm_90a only).  The .so is git-ignored: build() makes it."""
import os
import shutil
import subprocess

PKG_DIR = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(PKG_DIR, "csrc")
LIB_PATH = os.path.join(PKG_DIR, "libgmpi_mpi_render.so")
# the empty-space skipping kernels: a module of their own, loaded by the library on first use (the library's kernels keep their
# machine code)
SKIP_PATH = os.path.join(PKG_DIR, "libgmpi_mpi_render_skip.fatbin")
# the uint8-MPI kernels (GMPI_MPI_U8): likewise a module of their own
U8_PATH = os.path.join(PKG_DIR, "libgmpi_mpi_render_u8.fatbin")
SOURCES = ["mpi_render.cu"]
SKIP_SOURCES = ["mpi_skip.cu"]
U8_SOURCES = ["mpi_u8.cu"]
HEADERS = ["mpi_common.cuh", "mpi_fwd_staged.cuh", "mpi_fwd_direct.cuh", "mpi_bwd_box.cuh", "tma_utils.cuh",
           os.path.join("..", "..", "include", "gmpi_mpi_render.h")]
ARCH_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "-diag-suppress", "1886"]
NVCC_FLAGS = ARCH_FLAGS + ["-shared", "-Xcompiler", "-fPIC"]


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
    """Builds the library and the skipping and uint8 modules next to it; returns the library's path."""
    for path, sources in ((SKIP_PATH, SKIP_SOURCES), (U8_PATH, U8_SOURCES)):
        if force or is_stale(path):
            _nvcc(ARCH_FLAGS + ["-fatbin", "-o", path] + sources, verbose)
    if force or is_stale(LIB_PATH):
        _nvcc(NVCC_FLAGS + ["-o", LIB_PATH] + SOURCES, verbose)
    return LIB_PATH
