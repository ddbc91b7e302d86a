"""CPU checks of 8-bit RGBA MPIs (GMPI_MPI_U8): the exact conversion of all 256 codes in the host build, the option bit, the refusals
and plan reasons that need no GPU, the Python dispatch rule, the machine code of the uint8 kernels (mpi_u8.cu),
and the reference's plane-image conversion recorded in tests/golden/u8_planes.npz."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib
from ml_gmpi_b200.mpi import _check_unorm8, _unorm8_mpi
from conftest import ROOT
from testlib import KEY_AC, KEY_U8, lib, library_kernels, render_kernels

INVALID, UNSUPPORTED = 1, 3
U8 = 128


def exact_codes():
    return np.arange(256, dtype=np.uint8).astype(np.float32) / 255.0


def test_host_conversion_is_exact_for_every_code(lib):
    out = np.zeros(256, np.float32)
    _lib.check(lib.gmpi_debug_u8_codes_host(out.ctypes.data))
    assert np.array_equal(out.view(np.uint32), exact_codes().view(np.uint32))
    t = (torch.arange(256, dtype=torch.uint8).float() / 255).numpy()
    assert np.array_equal(out.view(np.uint32), t.view(np.uint32))
    assert np.array_equal(g.unorm8_to_float(torch.arange(256, dtype=torch.uint8)).numpy().view(np.uint32), out.view(np.uint32))
    # a plain multiply by RN(1/255) is not the conversion (why the kernels correct the quotient)
    mul = np.arange(256, dtype=np.float32) * np.float32(1 / 255)
    assert int((mul != out).sum()) == 126
    assert lib.gmpi_debug_u8_codes_host(None) == INVALID


def test_option_bit_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    m = re.search(r"#define GMPI_MPI_U8 (\d+)u", hdr)
    assert m and int(m.group(1)) == _lib.OPT_MPI_U8 == U8
    assert re.search(r"#define GMPI_ABI_VERSION 2\b", hdr)


def _buf():
    buf = (ctypes.c_float * 4096)()
    return buf, ctypes.addressof(buf)


def _desc(p, options=U8, **kw):
    f = dict(M=1, V=1, N=1, Ht=16, Wt=16, H=8, W=8, rgba=p, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p, color=p, depth=p, flags=p)
    f.update(kw)
    return _lib.make_desc(options=options, **{k: v for k, v in f.items() if v is not None})


def test_refusals_need_no_gpu(lib):
    buf, p = _buf()
    big = 1 << 20
    fwd = lambda d: lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d))
    # with GMPI_MPI_F16: invalid, on every entry point that takes the bit
    both = _desc(p, options=U8 | _lib.OPT_MPI_F16)
    assert fwd(both) == INVALID and b"exclusive" in lib.gmpi_last_error()
    assert lib.gmpi_mpi_render_host_ex(ctypes.byref(both), 0) == INVALID
    assert lib.gmpi_mpi_render_fwd_skip_ex(ctypes.byref(both), p, big) == INVALID
    assert lib.gmpi_mpi_occupancy_bytes(ctypes.byref(both)) == -INVALID
    assert lib.gmpi_mpi_build_occupancy(ctypes.byref(both), p, big) == INVALID
    # a factored MPI
    for fac in (dict(rgba=None, rgb=p, alpha=p), dict(rgba=None, rgb=p, alpha=p, bg_rgb=p)):
        d = _desc(p, **fac)
        assert fwd(d) == UNSUPPORTED and b"GMPI_MPI_U8" in lib.gmpi_last_error()
        assert lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0) == UNSUPPORTED
        assert lib.gmpi_mpi_render_fwd_skip_ex(ctypes.byref(d), p, big) == UNSUPPORTED
        assert lib.gmpi_mpi_occupancy_bytes(ctypes.byref(d)) == -UNSUPPORTED
        assert lib.gmpi_mpi_build_occupancy(ctypes.byref(d), p, big) == UNSUPPORTED
    # a transmittance output (training forward)
    d = _desc(p, transmittance=p)
    assert fwd(d) == UNSUPPORTED and b"GMPI_MPI_U8" in lib.gmpi_last_error()
    assert lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0) == UNSUPPORTED
    assert lib.gmpi_mpi_render_fwd_skip_ex(ctypes.byref(d), p, big) == UNSUPPORTED
    # the backward calls and the deterministic scratch query
    d = _desc(p, color=None, depth=None, g_color=p, g_rgba=p)
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == UNSUPPORTED and b"GMPI_MPI_U8" in lib.gmpi_last_error()
    assert lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), p, big) == UNSUPPORTED
    assert lib.gmpi_mpi_render_bwd_deterministic_scratch_bytes(ctypes.byref(d)) == -UNSUPPORTED
    # every classic entry point
    sizes = (1, 1, 1, 16, 16, 8, 8)
    calls = [lambda: lib.gmpi_mpi_render_fwd(*[p] * 9, *sizes, U8, None),
             lambda: lib.gmpi_mpi_render_fwd_train(*[p] * 10, *sizes, U8, None),
             lambda: lib.gmpi_mpi_render_fwd_gather(*[p] * 7, 1, 0, p, *sizes, U8, None),
             lambda: lib.gmpi_mpi_render_bwd(*[p] * 9, *sizes, U8, None),
             lambda: lib.gmpi_mpi_render_bwd_saved(*[p] * 10, *sizes, U8, None),
             lambda: lib.gmpi_mpi_render_fwd_host(*[p] * 9, *sizes, U8, 0)]
    for call in calls:
        assert call() == UNSUPPORTED and b"GMPI_MPI_U8" in lib.gmpi_last_error()
    # the map size of an expanded uint8 MPI is the fp32 MPI's
    for M, N, Ht, Wt in ((1, 1, 1, 1), (2, 3, 37, 300), (4, 96, 1024, 1024)):
        a, b = _desc(p, M=M, N=N, Ht=Ht, Wt=Wt), _desc(p, options=0, M=M, N=N, Ht=Ht, Wt=Wt)
        assert lib.gmpi_mpi_occupancy_bytes(ctypes.byref(a)) == lib.gmpi_mpi_occupancy_bytes(ctypes.byref(b)) > 0


def _plan(u8, Wt=1024, **ptrs):
    return _lib.fwd_plan(_lib.make_desc(options=U8 if u8 else 0, M=4, V=4, N=96, Ht=1024, Wt=Wt, H=1024, W=1024, **ptrs))


def test_plan_query_sees_the_dtype(lib):
    assert _plan(True) == (_lib.PLAN_STAGED, 0) and _plan(True, Wt=1008) == (_lib.PLAN_STAGED, 0)
    for Wt in (1016, 1020, 1022, 1000):          # rows of Wt bytes: 16-byte multiples only when Wt % 16 == 0
        assert _plan(False, Wt=Wt) == (_lib.PLAN_STAGED, 0) or Wt % 4
        assert _plan(True, Wt=Wt) == (_lib.PLAN_DIRECT, 1), Wt
    assert _plan(True, rgba=8) == (_lib.PLAN_DIRECT, 8) and _plan(True, rgba=4) == (_lib.PLAN_DIRECT, 8)
    assert _plan(True, rgba=16) == (_lib.PLAN_STAGED, 0)
    assert _plan(True, Wt=1020, rgba=8) == (_lib.PLAN_DIRECT, 9)


def test_python_dispatch_rule(lib):
    """Native uint8 only when the uint8 plan is the plan of a fresh fp32 allocation of the shape; otherwise the exact conversion."""
    u8 = lambda *s: torch.randint(0, 256, s, dtype=torch.uint8)
    rgba = u8(1, 2, 4, 8, 32)
    mpi, opts = _unorm8_mpi([rgba, None, None, None], 4, 1024, 1024, 1)
    assert opts == 1 | U8 and mpi[0].dtype == torch.uint8 and mpi[0].data_ptr() == rgba.data_ptr()
    narrow = u8(1, 2, 4, 8, 24)                   # Wt % 4 == 0, Wt % 16 != 0: staged in fp32, direct in uint8
    mpi, opts = _unorm8_mpi([narrow, None, None, None], 4, 1024, 1024, 1)
    assert opts == 1 and mpi[0].dtype == torch.float32
    assert np.array_equal(mpi[0].numpy(), narrow.numpy().astype(np.float32) / 255.0)
    mpi, opts = _unorm8_mpi([narrow, None, None, None], 1, 8, 8, 0)         # direct either way (few tiles): native
    assert opts == U8 and mpi[0].dtype == torch.uint8
    buf = torch.randint(0, 256, (2 * 4 * 8 * 32 + 32,), dtype=torch.uint8)
    off = (-buf.data_ptr()) % 16 + 8
    mis = buf[off:off + 2 * 4 * 8 * 32].view(1, 2, 4, 8, 32)     # 8 bytes past a 16-byte boundary
    mpi, opts = _unorm8_mpi([mis, None, None, None], 4, 1024, 1024, 0)
    assert opts == 0 and mpi[0].dtype == torch.float32
    t = u8(1, 2, 4, 32, 16).transpose(-1, -2)     # non-contiguous: rendered from a contiguous uint8 copy
    mpi, opts = _unorm8_mpi([t, None, None, None], 4, 1024, 1024, 0)
    assert opts == U8 and mpi[0].is_contiguous() and mpi[0].dtype == torch.uint8
    for bad in ([rgba.float(), None, None, None], [rgba.half(), None, None, None], [None, u8(1, 3, 8, 32), u8(1, 2, 1, 8, 32), None]):
        with pytest.raises(TypeError, match="uint8"):
            _check_unorm8(bad)


# ------------------------------------------------------------------------------------------------------------------------
# machine code of the uint8 kernels
# ------------------------------------------------------------------------------------------------------------------------
def test_u8_kernel_keys_of_the_library_and_resources():
    """8 staged kernels ([skip][align_corners][early stop]) with TMA loads and 8-bit shared-memory taps, 4 direct kernels, the map
    build and the conversion hook: at most 128 registers, no stack, no local memory, no spills."""
    g.build_library()
    funcs = {n: k for n, k in library_kernels().items() if (k.key or 0) & KEY_U8 or "u8" in k.template}
    staged = {**render_kernels(funcs, "mpi_fwd_staged_kernel"), **render_kernels(funcs, "mpi_fwd_skip_kernel")}
    direct = render_kernels(funcs, "mpi_fwd_direct_kernel")
    assert len(staged) == 8 and len(direct) == 4, sorted(funcs)
    assert {funcs[n].template for n in set(funcs) - set(staged) - set(direct)} == {"gmpi_occ_expanded_u8", "gmpi_u8_codes"}, sorted(funcs)
    for n, k in staged.items():
        b = k.sass
        assert "UTMALDG" in b and "SYNCS.PHASECHK.TRANS64.TRYWAIT" in b and "LDS.U8" in b, n
        assert " STL" not in b and " LDL" not in b, n
        assert (k.regs, k.stack, k.local) == (128, 0, 0), (n, k.regs, k.stack, k.local)
    for n, k in funcs.items():
        assert k.regs <= 128 and (k.stack, k.local) == (0, 0), (n, k.regs, k.stack, k.local)
    b = next(k.sass for k in direct.values() if k.key == KEY_U8 | KEY_AC)
    assert "LDG.E.U8" in b or "LDG.E.U8.CONSTANT" in b


# ------------------------------------------------------------------------------------------------------------------------
# the reference's conversion of RGBA8 plane images (oracle/make_golden_u8.py)
# ------------------------------------------------------------------------------------------------------------------------
def test_reference_plane_images_are_the_exact_conversion():
    """mpi_from_plane_imgs (mpi_utils.py:336-337) turns the seeded RGBA8 planes into the fp32 MPI the golden file recorded: bitwise
    unorm8_to_float of the planar uint8 tensor, and the host build of the kernels' conversion."""
    gd = np.load(os.path.join(ROOT, "tests", "golden", "u8_planes.npz"))
    u8, ref = gd["rgba_u8"], gd["rgba"]
    assert u8.dtype == np.uint8 and ref.dtype == np.float32 and u8.shape == ref.shape and u8.ndim == 5 and u8.shape[2] == 4
    assert np.array_equal(g.unorm8_to_float(torch.from_numpy(u8)).numpy().view(np.uint32), ref.view(np.uint32))
    assert np.array_equal((torch.from_numpy(u8).float() / 255).numpy().view(np.uint32), ref.view(np.uint32))
    codes = np.zeros(256, np.float32)
    g.build_library()
    _lib.check(_lib.load().gmpi_debug_u8_codes_host(codes.ctypes.data))
    assert np.array_equal(codes[u8].view(np.uint32), ref.view(np.uint32))
