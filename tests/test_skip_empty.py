"""CPU-side checks of the opt-in empty-space skipping (gmpi_mpi_build_occupancy, gmpi_mpi_render_fwd_skip_ex): the exports, the
map-size query, the refusals that need no GPU, the producer's box-versus-map test against a brute-force restatement, and the
resources of the skipping kernels (mpi_skip.cu: 128 registers, no spills).  test_library_build.py checks their machine code."""
import ctypes
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import ml_gmpi_b200 as g  # noqa: E402
from ml_gmpi_b200 import _lib  # noqa: E402
from testlib import KEY_U8, lib, library_kernels, render_kernels  # noqa: E402

ERR_INVALID, ERR_UNSUPPORTED = 1, 3
B = 8


def _buf():
    buf = (ctypes.c_float * 64)()
    return buf, ctypes.addressof(buf)


def _desc(p, *, M=1, V=1, N=2, Ht=4, Wt=4, H=4, W=4, factored=False, bg=False, **kw):
    """A forward descriptor whose pointers are host memory (never dereferenced: every call below is refused first)."""
    mpi = dict(rgb=p, alpha=p, bg_rgb=p if bg else None) if factored else dict(rgba=p)
    fields = dict(M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p, color=p, depth=p, flags=p, **mpi)
    fields.update(kw)
    return _lib.make_desc(**fields)


def occ_bytes_formula(M, N, Ht, Wt):
    """M*N planes of ceil(Ht/8) block rows of ceil(ceil(Wt/8)/32) 32-bit words."""
    return M * N * -(-Ht // B) * -(-(-(-Wt // B)) // 32) * 4


def test_symbols_are_exported(lib):
    for s in ("gmpi_mpi_occupancy_bytes", "gmpi_mpi_build_occupancy", "gmpi_mpi_render_fwd_skip_ex", "gmpi_debug_fwd_skip_stats",
              "gmpi_debug_box_occupied"):
        assert hasattr(lib, s) and s in _lib.EXPORTS, s


@pytest.mark.parametrize("factored,bg,f16", [(False, False, False), (False, False, True), (True, False, False), (True, True, True)])
@pytest.mark.parametrize("M,N,Ht,Wt", [(1, 1, 1, 1), (2, 3, 5, 7), (4, 96, 1024, 1024), (3, 17, 37, 300), (1, 2, 8, 256), (1, 2, 9, 257)])
def test_map_size_query_matches_the_layout(lib, factored, bg, f16, M, N, Ht, Wt):
    buf, p = _buf()
    d = _desc(p, M=M, N=N, Ht=Ht, Wt=Wt, factored=factored, bg=bg, options=_lib.OPT_MPI_F16 if f16 else 0)
    assert lib.gmpi_mpi_occupancy_bytes(ctypes.byref(d)) == occ_bytes_formula(M, N, Ht, Wt)
    assert _lib.occupancy_bytes(d) == occ_bytes_formula(M, N, Ht, Wt)


def test_map_of_the_head_case_is_small():
    """4 MPIs x 96 planes x 1024^2: 128 x 4 words per plane, 768 KiB in all (1/2048 of the fp32 MPI)."""
    assert occ_bytes_formula(4, 96, 1024, 1024) == 4 * 96 * 128 * 4 * 4 == 786432


def test_refusals_need_no_gpu(lib):
    buf, p = _buf()
    occ = (ctypes.c_uint32 * 64)()
    o = ctypes.addressof(occ)
    big = 1 << 40
    assert lib.gmpi_mpi_occupancy_bytes(None) == -ERR_INVALID
    assert lib.gmpi_mpi_occupancy_bytes(ctypes.byref(_desc(p, N=0))) == -ERR_INVALID and b"bad sizes" in lib.gmpi_last_error()
    assert lib.gmpi_mpi_occupancy_bytes(ctypes.byref(_desc(p, rgba=None))) == -ERR_INVALID and b"null input" in lib.gmpi_last_error()
    for fn in (lib.gmpi_mpi_build_occupancy, lib.gmpi_mpi_render_fwd_skip_ex):
        assert fn(None, o, big) == ERR_INVALID and b"null descriptor" in lib.gmpi_last_error()
        d = _desc(p)
        assert fn(ctypes.byref(d), None, big) == ERR_INVALID and b"null occupancy" in lib.gmpi_last_error()
        assert fn(ctypes.byref(d), o + 2, big) == ERR_INVALID and b"4-byte aligned" in lib.gmpi_last_error()
        need = occ_bytes_formula(1, 2, 4, 4)
        assert fn(ctypes.byref(d), o, need - 1) == ERR_INVALID and b"smaller than" in lib.gmpi_last_error()
        assert str(need).encode() in lib.gmpi_last_error()
        bad = _desc(p, factored=True, alpha=None)
        assert fn(ctypes.byref(bad), o, big) == ERR_INVALID and b"null input" in lib.gmpi_last_error()
    call = lambda d: lib.gmpi_mpi_render_fwd_skip_ex(ctypes.byref(d), o, big)
    assert call(_desc(p, transmittance=p)) == ERR_UNSUPPORTED and b"forward-only" in lib.gmpi_last_error()
    # what gmpi_mpi_render_fwd_ex refuses, this call refuses with the same code
    for bad in (_desc(p, view2mpi=None), _desc(p, V=3, view_group=2), _desc(p, options=_lib.OPT_EARLY_STOP, early_stop=1.5)):
        assert call(bad) == lib.gmpi_mpi_render_fwd_ex(ctypes.byref(bad)) == ERR_INVALID
    assert lib.gmpi_debug_fwd_skip_stats(None, None) == ERR_INVALID


# ------------------------------------------------------------------------------------------------------------------------
# the producer's box-versus-map test (gmpi_debug_box_occupied: the kernel's code, evaluated on the host)
# ------------------------------------------------------------------------------------------------------------------------
def _plane_map(occupied_blocks):
    """[rows, cols] bool block grid -> the plane's map words [rows, words] (bit b of word w = block column 32 w + b)."""
    rows, cols = occupied_blocks.shape
    words = -(-cols // 32)
    out = np.zeros((rows, words), np.uint32)
    for r, c in zip(*np.nonzero(occupied_blocks)):
        out[r, c // 32] |= np.uint32(1 << (c % 32))
    return out


def _brute(occupied_blocks, Ht, Wt, bx0, by0, bw, rows):
    """Any occupied block under a texel of [bx0, bx0 + bw) x [by0, by0 + rows) inside the texture."""
    x0, x1, y0, y1 = max(bx0, 0), min(bx0 + bw - 1, Wt - 1), max(by0, 0), min(by0 + rows - 1, Ht - 1)
    if x0 > x1 or y0 > y1:
        return False
    return bool(occupied_blocks[y0 // B: y1 // B + 1, x0 // B: x1 // B + 1].any())


def _query(lib, words, Ht, Wt, bx0, by0, bw, rows):
    return lib.gmpi_debug_box_occupied(words.ctypes.data, Ht, Wt, bx0, by0, bw, rows)


@pytest.mark.parametrize("Ht,Wt", [(64, 64), (37, 83), (300, 520), (1024, 1024)])
def test_box_test_matches_brute_force_on_single_blocks(lib, Ht, Wt):
    """One occupied block at a time, boxes of the staged widths and heights whose edges lie on, just before and just after that
    block's edges (and the texture's partial edge blocks): the test reports exactly the boxes that cover it, so it never reports
    "empty" for a box over an occupied block, and never keeps a stage whose blocks are all empty."""
    rows_b, cols_b = -(-Ht // B), -(-Wt // B)
    targets = {(0, 0), (rows_b - 1, cols_b - 1), (rows_b // 2, cols_b // 2), (0, cols_b - 1), (rows_b - 1, 0)}
    if cols_b > 32:
        targets |= {(1, 31), (1, 32), (rows_b // 3, 63 if cols_b > 63 else cols_b - 1)}
    widths = [56, 64, 72, 80, 88, 96]
    heights = [4, 8, 20, 32, 44]
    for (tr, tc) in targets:
        occ = np.zeros((rows_b, cols_b), bool)
        occ[tr, tc] = True
        words = np.ascontiguousarray(_plane_map(occ))
        xs = sorted({tc * B + d for d in (-100, -89, -88, -9, -8, -7, -1, 0, 1, 7, 8, 9)} | {-200, -4, Wt - 1, Wt, Wt + 4})
        ys = sorted({tr * B + d for d in (-45, -44, -9, -8, -7, -1, 0, 1, 7, 8, 9)} | {-50, -2, Ht - 1, Ht})
        for bw in widths:
            for rows in heights:
                for bx0 in xs:
                    for by0 in ys:
                        got = _query(lib, words, Ht, Wt, bx0, by0, bw, rows)
                        assert got == int(_brute(occ, Ht, Wt, bx0, by0, bw, rows)), (tr, tc, bx0, by0, bw, rows)


def test_box_test_matches_brute_force_on_random_maps(lib):
    rng = np.random.default_rng(3)
    for trial in range(40):
        Ht, Wt = int(rng.integers(1, 700)), int(rng.integers(1, 700))
        occ = rng.random((-(-Ht // B), -(-Wt // B))) < rng.choice([0.002, 0.02, 0.2])
        words = np.ascontiguousarray(_plane_map(occ))
        for _ in range(300):
            bw, rows = int(rng.choice([56, 64, 72, 80, 88, 96])), int(rng.choice([4, 12, 24, 36, 44]))
            bx0, by0 = int(rng.integers(-100, Wt + 10)) & ~3, int(rng.integers(-50, Ht + 10))
            assert _query(lib, words, Ht, Wt, bx0, by0, bw, rows) == int(_brute(occ, Ht, Wt, bx0, by0, bw, rows))


def test_box_test_refuses_bad_arguments(lib):
    w = np.zeros(4, np.uint32)
    assert lib.gmpi_debug_box_occupied(None, 8, 8, 0, 0, 8, 8) < 0
    assert _query(lib, w, 0, 8, 0, 0, 8, 8) < 0 and _query(lib, w, 8, 8, 0, 0, 0, 8) < 0


# ------------------------------------------------------------------------------------------------------------------------
# resources of the skipping kernels
# ------------------------------------------------------------------------------------------------------------------------
def test_skip_kernel_keys_of_the_library_use_128_registers_without_spills():
    g.build_library()
    kernels = library_kernels()
    res = {n: (k.regs, k.stack, k.local) for n, k in kernels.items()}
    fwd = {n: res[n] for n in render_kernels(kernels, "mpi_fwd_skip_kernel", lacks=KEY_U8)}
    occ = {n: r for n, r in res.items() if n.startswith("gmpi_occ_") and not n.endswith("_u8")}
    assert len(fwd) == 16 and set(occ) == {
        "gmpi_occ_expanded_f32", "gmpi_occ_expanded_f16", "gmpi_occ_factored_f32", "gmpi_occ_factored_f16"}, sorted(res)
    assert all(r == (128, 0, 0) for r in fwd.values()), fwd
    assert all(r[1:] == (0, 0) for r in occ.values()), occ
