"""CPU-side checks of the deterministic backward (gmpi_mpi_render_bwd_deterministic_ex): the scratch-size query, the refusals
that need no GPU, and the choice of the fixed-point fraction bits k (no int64 sum can wrap).  test_library_build.py checks the
machine code of its kernels."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from ml_gmpi_b200 import _lib  # noqa: E402
from testlib import lib  # noqa: E402

ERR_INVALID, ERR_UNSUPPORTED = 1, 3


def _buf():
    buf = (ctypes.c_float * 64)()
    return buf, ctypes.addressof(buf)


def _desc(p, *, M=1, V=1, N=2, Ht=4, Wt=4, H=4, W=4, factored=False, bg=False, **kw):
    """A backward descriptor whose pointers are host memory (never dereferenced: every call below is refused first)."""
    mpi = dict(rgb=p, alpha=p, bg_rgb=p if bg else None, g_rgb=p, g_alpha=p, g_bg_rgb=p if bg else None) if factored \
        else dict(rgba=p, g_rgba=p)
    fields = dict(M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p, g_color=p, **mpi)
    fields.update(kw)
    return _lib.make_desc(**fields)


def scratch_bytes_formula(M, N, Ht, Wt, factored, bg):
    """The scratch layout of the header: 256 bytes, an int64 sum per gradient element, four non-finite bits per element."""
    tex = Ht * Wt
    G = (M * 3 * tex + M * N * tex + (M * 3 * tex if bg else 0)) if factored else M * N * 4 * tex
    return 256 + 8 * G + 4 * ((G + 7) // 8)


def ceil_log2(x):
    return max(0, int(x - 1).bit_length())


def fix_bits(H, W, V, planes):
    """k of the unit 2^(E - k): one (view, plane) gives a texel at most H*W taps, V bounds the views of an MPI."""
    return 61 - ceil_log2(H * W) - ceil_log2(V) - ceil_log2(planes)


@pytest.mark.parametrize("factored,bg", [(False, False), (True, False), (True, True)])
@pytest.mark.parametrize("M,N,Ht,Wt", [(1, 1, 1, 1), (2, 3, 5, 7), (4, 96, 1024, 1024), (3, 17, 64, 36)])
def test_scratch_size_query_matches_the_layout(lib, factored, bg, M, N, Ht, Wt):
    buf, p = _buf()
    d = _desc(p, M=M, N=N, Ht=Ht, Wt=Wt, factored=factored, bg=bg)
    assert lib.gmpi_mpi_render_bwd_deterministic_scratch_bytes(ctypes.byref(d)) == scratch_bytes_formula(M, N, Ht, Wt, factored, bg)
    assert _lib.deterministic_scratch_bytes(d) == scratch_bytes_formula(M, N, Ht, Wt, factored, bg)


def test_scratch_size_of_the_training_shape():
    """4 MPIs x 96 planes x 1024^2: 13.7 GB expanded, 3.6 GB factored with bg_rgb (8 B per gradient element + its non-finite bits)."""
    assert scratch_bytes_formula(4, 96, 1024, 1024, False, False) == 256 + 8.5 * 4 * 96 * 4 * 1024 ** 2
    assert round(scratch_bytes_formula(4, 96, 1024, 1024, True, True) / 1e9, 1) == 3.6


def test_scratch_size_query_refuses_bad_descriptors(lib):
    assert lib.gmpi_mpi_render_bwd_deterministic_scratch_bytes(None) == -ERR_INVALID
    buf, p = _buf()
    d = _desc(p, N=0)
    assert lib.gmpi_mpi_render_bwd_deterministic_scratch_bytes(ctypes.byref(d)) == -ERR_INVALID
    assert b"bad sizes" in lib.gmpi_last_error()
    d = _desc(p)
    d.struct_bytes = 8
    assert lib.gmpi_mpi_render_bwd_deterministic_scratch_bytes(ctypes.byref(d)) == -ERR_INVALID
    with pytest.raises(_lib.GmpiLibraryError, match="struct_bytes"):
        _lib.deterministic_scratch_bytes(d)


def test_refusals_need_no_gpu(lib):
    buf, p = _buf()
    scratch = (ctypes.c_uint64 * 16)()
    s = (ctypes.addressof(scratch) + 15) & ~15
    big = 1 << 40
    call = lambda d, ptr, n: lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), ptr, n)
    assert lib.gmpi_mpi_render_bwd_deterministic_ex(None, s, big) == ERR_INVALID and b"null descriptor" in lib.gmpi_last_error()
    d = _desc(p)
    assert call(d, None, big) == ERR_INVALID and b"null scratch" in lib.gmpi_last_error()
    need = scratch_bytes_formula(1, 2, 4, 4, False, False)
    assert call(d, s, need - 1) == ERR_INVALID and b"smaller than" in lib.gmpi_last_error()
    assert str(need).encode() in lib.gmpi_last_error()
    assert call(d, s + 8, big) == ERR_INVALID and b"16-byte aligned" in lib.gmpi_last_error()
    assert call(_desc(p, options=_lib.OPT_MPI_F16), s, big) == ERR_UNSUPPORTED and b"forward-only" in lib.gmpi_last_error()
    assert call(_desc(p, options=_lib.OPT_EARLY_STOP), s, big) == ERR_UNSUPPORTED and b"forward-only" in lib.gmpi_last_error()
    assert call(_desc(p, cam=p), s, big) == ERR_UNSUPPORTED and b"cam is forward-only" in lib.gmpi_last_error()
    # what gmpi_mpi_render_bwd_ex refuses, this call refuses with the same code
    for bad in (_desc(p, g_color=None), _desc(p, factored=True, bg=True, g_bg_rgb=None), _desc(p, V=3, view_group=2)):
        assert call(bad, s, big) == lib.gmpi_mpi_render_bwd_ex(ctypes.byref(bad)) == ERR_INVALID


def test_fraction_bits_refusal_is_at_the_restated_edge(lib):
    """k >= 24 is required; the library's k is the restated one: 4096^2 pixels and 8192 views leave k = 24 for a single plane, one
    more view (or a factored MPI's colour summing two planes) leaves 23 and is refused."""
    assert fix_bits(4096, 4096, 8192, 1) == 24 and fix_bits(4096, 4096, 8193, 1) == 23 and fix_bits(4096, 4096, 8192, 2) == 23
    buf, p = _buf()
    scratch = (ctypes.c_uint64 * 16)()
    s = (ctypes.addressof(scratch) + 15) & ~15
    for d in (_desc(p, V=8193, H=4096, W=4096), _desc(p, V=8192, H=4096, W=4096, factored=True)):
        assert lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), s, 1 << 62) == ERR_UNSUPPORTED
        assert b"23 fraction bits" in lib.gmpi_last_error()


def _worst_case_sum(H, W, V, planes):
    """The largest |sum| of one element in units 2^(E - k): C = H*W*V*planes taps, each below 2^k w + max(1/2, the box's rounding
    2^(k-23) in these units) with weights w <= 1, plus 1/2 per tile flush (at most one per tap)."""
    k = fix_bits(H, W, V, planes)
    C = H * W * V * planes
    return 2 ** k * C + C * max(0.5, 2.0 ** (k - 23)) + 0.5 * C


def test_worst_case_sums_cannot_wrap_int64():
    rng = np.random.default_rng(0)
    shapes = [(1, 1, 1, 1), (1024, 1024, 4, 1), (1024, 1024, 4, 96), (256, 256, 256, 32), (512, 512, 15, 96), (4096, 4096, 8192, 1)]
    shapes += [tuple(int(x) for x in (rng.integers(1, 8193), rng.integers(1, 8193), rng.integers(1, 4097), rng.integers(1, 1025)))
               for _ in range(500)]
    for H, W, V, P in shapes:
        if fix_bits(H, W, V, P) < 24:
            continue                                # refused by the library
        assert _worst_case_sum(H, W, V, P) < 2 ** 63, (H, W, V, P)
