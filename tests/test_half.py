"""CPU checks of fp16 MPIs (GMPI_MPI_F16): the option bit, the refusals and plan reasons that need no GPU, the Python dispatch
rule, and the machine code of the fp16 staged kernels."""
import ctypes
import os
import re

import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib
from ml_gmpi_b200.mpi import _half_mpi
from conftest import ROOT
from testlib import KEY_F16, lib, library_kernels, render_kernels

UNSUPPORTED = 3


def test_option_bit_matches_the_header():
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    m = re.search(r"#define GMPI_MPI_F16 (\d+)u", hdr)
    assert m and int(m.group(1)) == _lib.OPT_MPI_F16 == 64
    assert re.search(r"#define GMPI_ABI_VERSION 2\b", hdr)


def _buf():
    buf = (ctypes.c_float * 4096)()
    return buf, ctypes.addressof(buf)


def test_refusals_need_no_gpu(lib):
    buf, p = _buf()
    f16 = _lib.OPT_MPI_F16
    # with a transmittance output (training forward), on the device and the host entry points
    d = _lib.make_desc(options=f16, M=1, V=1, N=1, Ht=8, Wt=8, H=8, W=8, rgba=p, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p,
                       color=p, depth=p, flags=p, transmittance=p)
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == UNSUPPORTED and b"GMPI_MPI_F16" in lib.gmpi_last_error()
    assert lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0) == UNSUPPORTED and b"GMPI_MPI_F16" in lib.gmpi_last_error()
    # the backward
    d = _lib.make_desc(options=f16, M=1, V=1, N=1, Ht=8, Wt=8, H=8, W=8, rgba=p, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p,
                       g_color=p, g_rgba=p)
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == UNSUPPORTED and b"GMPI_MPI_F16" in lib.gmpi_last_error()
    # every classic entry point
    sizes = (1, 1, 1, 8, 8, 8, 8)
    calls = [lambda: lib.gmpi_mpi_render_fwd(*[p] * 9, *sizes, f16, None),
             lambda: lib.gmpi_mpi_render_fwd_train(*[p] * 10, *sizes, f16, None),
             lambda: lib.gmpi_mpi_render_fwd_gather(*[p] * 7, 1, 0, p, *sizes, f16, None),
             lambda: lib.gmpi_mpi_render_bwd(*[p] * 9, *sizes, f16, None),
             lambda: lib.gmpi_mpi_render_bwd_saved(*[p] * 10, *sizes, f16, None),
             lambda: lib.gmpi_mpi_render_fwd_host(*[p] * 9, *sizes, f16, 0)]
    for call in calls:
        assert call() == UNSUPPORTED and b"GMPI_MPI_F16" in lib.gmpi_last_error()


def _plan(lib, half, Wt=1024, **ptrs):
    return _lib.fwd_plan(_lib.make_desc(options=_lib.OPT_MPI_F16 if half else 0, M=4, V=4, N=96, Ht=1024, Wt=Wt, H=1024, W=1024, **ptrs))


def test_plan_query_sees_the_dtype(lib):
    assert _plan(lib, False) == (_lib.PLAN_STAGED, 0) and _plan(lib, True) == (_lib.PLAN_STAGED, 0)
    assert _plan(lib, False, Wt=1020) == (_lib.PLAN_STAGED, 0)         # fp32 rows of 4080 B are 16-byte multiples
    assert _plan(lib, True, Wt=1020) == (_lib.PLAN_DIRECT, 1)          # fp16 rows of 2040 B are not
    assert _plan(lib, True, Wt=1022) == (_lib.PLAN_DIRECT, 1)
    assert _plan(lib, True, rgba=8) == (_lib.PLAN_DIRECT, 8)
    assert _plan(lib, True, rgb=16, alpha=32, bg_rgb=40) == (_lib.PLAN_DIRECT, 8)
    assert _plan(lib, True, rgb=16, alpha=32, bg_rgb=48) == (_lib.PLAN_STAGED, 0)
    # the classic plan query agrees for fp32
    why = ctypes.c_uint32(0)
    assert lib.gmpi_mpi_render_fwd_plan(4, 96, 1024, 1020, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_STAGED
    d = _lib.make_desc(M=1, V=1, N=1, Ht=8, Wt=8, H=8, W=8)
    d.struct_bytes = 8
    with pytest.raises(_lib.GmpiLibraryError, match="struct_bytes"):
        _lib.fwd_plan(d)


def test_python_dispatch_rule(lib):
    """Native fp16 only when every MPI tensor is fp16, autograd does not record for them and the plan is the fp32 plan."""
    half = lambda *s: torch.rand(s).half()
    rgba = half(1, 2, 4, 8, 16)
    got = _half_mpi([rgba, None, None, None], 4, 1024, 1024, 0)
    assert got is not None and got[0].dtype == torch.float16 and got[0].data_ptr() == rgba.data_ptr()
    assert _half_mpi([rgba.float(), None, None, None], 4, 1024, 1024, 0) is None
    rgb, alpha, bg = half(1, 3, 8, 16), half(1, 2, 1, 8, 16), half(1, 3, 8, 16)
    assert _half_mpi([None, rgb, alpha, bg], 4, 1024, 1024, 0) is not None
    assert _half_mpi([None, rgb, alpha, bg.float()], 4, 1024, 1024, 0) is None          # mixed dtypes: upcast
    narrow = half(1, 2, 4, 8, 12)                  # Wt % 4 == 0, Wt % 8 != 0: staged in fp32, direct in fp16
    assert _half_mpi([narrow, None, None, None], 4, 1024, 1024, 0) is None
    assert _half_mpi([narrow, None, None, None], 1, 8, 8, 0) is not None                 # direct either way (few tiles)
    grad = rgba.clone().requires_grad_(True)
    assert _half_mpi([grad, None, None, None], 4, 1024, 1024, 0) is None
    with torch.no_grad():
        got = _half_mpi([grad, None, None, None], 4, 1024, 1024, 0)
    assert got is not None and not got[0].requires_grad       # detached: the native path has no backward
    t = half(1, 2, 4, 16, 8).transpose(-1, -2)        # non-contiguous: rendered from a contiguous fp16 copy
    got = _half_mpi([t, None, None, None], 4, 1024, 1024, 0)
    assert got is not None and got[0].is_contiguous() and got[0].dtype == torch.float16


def test_sass_of_the_fp16_staged_kernel_keys():
    """The fp16 staged kernels are TMA + mbarrier kernels like the fp32 ones: 128 registers, no local memory, their taps are
    16-bit shared loads converted to fp32 (checked on the machine code, no GPU needed)."""
    g.build_library()
    funcs = library_kernels()
    kernels = render_kernels(funcs, "mpi_fwd_staged_kernel", has=KEY_F16)
    assert len(kernels) == 8, sorted(kernels)          # [early stop][align_corners][factored]; no training instantiation
    for n, k in kernels.items():
        b = k.sass
        assert "UTMALDG" in b and "SYNCS.PHASECHK.TRANS64.TRYWAIT" in b and "SYNCS.ARRIVE.TRANS64" in b, n
        assert "LDS.U16" in b and len(re.findall(r"\bFFMA\b", b)) > 200, n
        assert " STL" not in b and " LDL" not in b, n
        assert (k.regs, k.stack, k.local) == (128, 0, 0), (n, k.regs, k.stack, k.local)
    assert len(render_kernels(funcs, "mpi_fwd_direct_kernel", has=KEY_F16)) == 4
    assert "_ZN4gmpi22mpi_check_range_kernelI6__half5uint4EEvPKT0_mmPj" in funcs     # mpi_check_range_kernel<__half, uint4>
