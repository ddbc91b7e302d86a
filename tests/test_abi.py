"""CPU-side checks of the drop-in boundary: the C-ABI library builds for sm_90a, loads, exports every
symbol include/gmpi_mpi_render.h declares, and validates arguments without touching a GPU."""
import ctypes
import os
import re

import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib
from conftest import ROOT
from testlib import KEY_AC, KEY_BWD, KEY_ES, KEY_F16, KEY_FAC, KEY_STAGED, KEY_U8, lib, library_kernels, render_kernels


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(gmpi_[a-z0-9_]+)\s*\(", hdr)))


C_TYPES = {"int": ctypes.c_int, "uint32_t": ctypes.c_uint32, "size_t": ctypes.c_size_t, "long long": ctypes.c_longlong}


def _ctype(decl):
    """The ctypes type of a C parameter or return declaration (its name, if any, dropped)."""
    if "*" in decl:
        if "gmpi_render_desc" in decl:
            return ctypes.POINTER(_lib.RenderDesc)
        return ctypes.c_char_p if re.match(r"(const\s+)?char\s*\*$", decl) else ctypes.c_void_p
    return C_TYPES[decl if decl in C_TYPES else decl.rsplit(" ", 1)[0]]


def declared_prototypes():
    """{name: (return declaration, [parameter declarations])} of every function the header declares."""
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    out = {}
    for ret, name, params in re.findall(r"^([a-z][a-z ]*?\**)\s*(gmpi_[a-z0-9_]+)\s*\(([^)]*)\)\s*;", hdr, re.M):
        params = " ".join(params.split())
        out[name] = (ret.strip(), [] if params == "void" else [p.strip() for p in params.split(",")])
    return out


def test_header_symbols_are_exported(lib):
    syms = declared_symbols()
    assert "gmpi_mpi_render_fwd" in syms and "gmpi_mpi_render_bwd" in syms
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in the header but not exported"
    assert sorted(_lib.EXPORTS) == syms
    # every exported function has a signature that matches its prototype: ctypes' defaults (an int return, int arguments) would
    # cut 64-bit pointers short
    protos = declared_prototypes()
    assert list(_lib.SIGNATURES) == list(protos)              # the header's order
    for name, (restype, argtypes) in _lib.SIGNATURES.items():
        ret, params = protos[name]
        assert restype is _ctype(ret), (name, ret)
        assert len(argtypes) == len(params), (name, params)
        for i, (t, p) in enumerate(zip(argtypes, params)):
            assert t is _ctype(p), (name, i, p)


def test_abi_version_and_constants(lib):
    assert lib.gmpi_abi_version() == _lib.ABI_VERSION
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    for name, val in [("GMPI_FLAG_RGBA_RANGE", _lib.FLAG_RGBA_RANGE), ("GMPI_FLAG_ALPHA_RANGE", _lib.FLAG_ALPHA_RANGE),
                      ("GMPI_FLAG_LAST_PLANE_OOB", _lib.FLAG_LAST_PLANE_OOB),
                      ("GMPI_FLAG_PLANE_BEHIND_EYE", _lib.FLAG_PLANE_BEHIND_EYE),
                      ("GMPI_ALIGN_CORNERS", _lib.OPT_ALIGN_CORNERS), ("GMPI_CHECK_LAST_PLANE", _lib.OPT_CHECK_LAST_PLANE),
                      ("GMPI_COLOR_MINUS1_1", _lib.OPT_COLOR_MINUS1_1), ("GMPI_ZERO_GRAD", _lib.OPT_ZERO_GRAD)]:
        m = re.search(rf"#define {name} (\d+)u", hdr)
        assert m and int(m.group(1)) == val, name


def test_argument_validation_needs_no_gpu(lib):
    rc = lib.gmpi_mpi_render_fwd(None, None, None, None, None, None, None, None, None, 1, 1, 1, 1, 1, 1, 1, 0, None)
    assert rc == 1 and b"null" in lib.gmpi_last_error()
    buf = (ctypes.c_float * 16)()
    p = ctypes.addressof(buf)
    rc = lib.gmpi_mpi_render_fwd(p, p, p, p, p, p, p, p, p, 1, 1, 0, 4, 4, 4, 4, 0, None)
    assert rc == 1 and b"bad sizes" in lib.gmpi_last_error()
    rc = lib.gmpi_mpi_render_bwd(p, p, p, p, p, p, None, None, None, 1, 1, 1, 4, 4, 4, 4, 0, None)
    assert rc == 1


def test_ring_depth_hooks_validate_without_gpu(lib):
    for bad in (-1, 1, 4):
        assert lib.gmpi_debug_set_fwd_stages(bad) == 1 and b"stages must be" in lib.gmpi_last_error()
    for ok in (2, 3, 0):                        # ends on auto
        assert lib.gmpi_debug_set_fwd_stages(ok) == 0
    assert lib.gmpi_debug_fwd_ring_stages(1, 1, 0, 64, 64, 1) < 0
    assert lib.gmpi_debug_fwd_ring_stages(1, 1, 8, 64, 64, -1) < 0


def test_cubin_is_sm90a():
    import subprocess
    out = subprocess.run(["cuobjdump", "-lelf", g._build.LIB_PATH], capture_output=True, text=True).stdout
    assert "sm_90a" in out, out


def test_no_cpu_fallback():
    mpi = g.MPI(align_corners=True)
    rgba = torch.rand(1, 2, 4, 8, 8)
    dhw = torch.tensor([[[1.0, 0.2, 0.2], [1.1, 0.2, 0.2]]])
    ray = torch.zeros(1, 3, 4, 4); ray[:, 2] = 1
    with pytest.raises(RuntimeError, match="CUDA devices only"):
        mpi(batch_rgba=rgba, batch_dhw=dhw, batch_ray_dir=[ray], batch_eye_pos=[torch.zeros(1, 3)],
            batch_z_dir=[torch.tensor([[0., 0., 1.]])], separate_background=None)


def test_shape_asserts_match_reference_messages():
    mpi = g.MPI()
    ray = torch.zeros(1, 3, 4, 4)
    with pytest.raises(AssertionError, match="Expected rgba to be of shape"):
        mpi(batch_rgba=torch.rand(1, 2, 3, 8, 8), batch_dhw=torch.rand(1, 2, 3), batch_ray_dir=[ray],
            batch_eye_pos=[torch.zeros(1, 3)], batch_z_dir=[torch.zeros(1, 3)], separate_background=None)
    with pytest.raises(AssertionError, match="Expected dhw to be of shape"):
        mpi(batch_rgba=torch.rand(1, 2, 4, 8, 8), batch_dhw=torch.rand(1, 3, 3), batch_ray_dir=[ray],
            batch_eye_pos=[torch.zeros(1, 3)], batch_z_dir=[torch.zeros(1, 3)], separate_background=None)
    with pytest.raises(AssertionError, match="Expected ray_dir to be of shape"):
        mpi(batch_rgba=torch.rand(1, 2, 4, 8, 8), batch_dhw=torch.rand(1, 2, 3), batch_ray_dir=[ray[0]],
            batch_eye_pos=[torch.zeros(1, 3)], batch_z_dir=[torch.zeros(1, 3)], separate_background=None)


def test_pack_views_is_mpi_major():
    rays = [torch.zeros(2, 3, 4, 4), torch.ones(1, 3, 4, 4), torch.zeros(3, 3, 4, 4)]
    eyes = [torch.zeros(2, 3), torch.ones(1, 3), torch.zeros(3, 3)]
    v2m, ray, eye, z = g.MPI.pack_views(rays, eyes, eyes, torch.device("cpu"))
    assert v2m.tolist() == [0, 0, 1, 2, 2, 2] and v2m.dtype == torch.int32
    assert ray.shape == (6, 3, 4, 4) and float(ray[2].min()) == 1.0


def test_plan_query_needs_no_gpu(lib):
    why = ctypes.c_uint32(0)
    assert lib.gmpi_mpi_render_fwd_plan(4, 96, 1024, 1024, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_STAGED and why.value == 0
    assert lib.gmpi_mpi_render_fwd_plan(4, 96, 1022, 1022, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 1
    assert lib.gmpi_mpi_render_fwd_plan(1, 16, 64, 64, 48, 48, None, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 2
    assert lib.gmpi_mpi_render_fwd_plan(4, 600, 1024, 1024, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 4
    assert lib.gmpi_mpi_render_fwd_plan(4, 96, 1024, 1024, 1024, 1024, 8, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 8


def test_render_desc_matches_header():
    """ctypes mirror of gmpi_render_desc: same fields, same order, pointer-sized where the header has pointers."""
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    body = re.search(r"typedef struct gmpi_render_desc \{(.*?)\} gmpi_render_desc;", hdr, re.S).group(1)
    names = re.findall(r"\b([a-zA-Z_0-9]+)(?:,|;)", body)
    assert [f[0] for f in _lib.RenderDesc._fields_] == names
    d = _lib.make_desc(M=1, V=2, options=5)
    assert d.struct_bytes == ctypes.sizeof(_lib.RenderDesc) and d.M == 1 and d.V == 2 and d.options == 5 and not d.rgba


def test_descriptor_entry_points_validate_without_gpu(lib):
    assert lib.gmpi_mpi_render_fwd_ex(None) == 1 and b"null descriptor" in lib.gmpi_last_error()
    d = _lib.make_desc(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4)
    d.struct_bytes = 8
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"struct_bytes" in lib.gmpi_last_error()
    d = _lib.make_desc(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4)
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"null input" in lib.gmpi_last_error()
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    # factored form needs both rgb and alpha; rgba and alpha together are rejected
    d = _lib.make_desc(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4, rgba=p, alpha=p, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p)
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1
    # backward with cam is unsupported (fast mode is forward-only)
    d = _lib.make_desc(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4, rgba=p, view2mpi=p, dhw=p, cam=p, g_color=p, g_rgba=p)
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == 3
    d = _lib.make_desc(M=1, V=3, N=1, Ht=4, Wt=4, H=4, W=4, view_group=2, rgba=p, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p)
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"view_group" in lib.gmpi_last_error()


def test_sass_of_the_hot_kernel_keys_is_tma_mbarrier_packed_math():
    """The shipped library's staged kernels are what DESIGN.md says they are (checked on the machine code, no GPU needed):
    TMA tensor loads + mbarrier transactions + the pixel-pair arithmetic as scalar FFMA in the forward (sm_90 has no packed
    fp32 instructions), additionally native integer shared atomics
    and vector global reductions in the backward; no local-memory spills in the expanded instantiations."""
    import re
    g.build_library()
    kernels = library_kernels()
    fwd = render_kernels(kernels, "mpi_fwd_staged_kernel", lacks=KEY_ES | KEY_F16 | KEY_U8)
    bwd = render_kernels(kernels, "mpi_bwd_box_kernel")
    assert len(fwd) == 8 and len(bwd) == 4                       # align_corners x training x factored; align_corners x factored
    for n, k in fwd.items():
        b = k.sass
        assert "UTMALDG" in b and "SYNCS.PHASECHK.TRANS64.TRYWAIT" in b and "SYNCS.ARRIVE.TRANS64" in b
        # 2 pairs x 16 taps x 2 loads per tap pair, for each box width: two in the factored ring, five in the expanded one
        widths = 2 if k.key & KEY_FAC else 5
        assert len(re.findall(r"\bFFMA\b", b)) > 200 and b.count("LDS") >= 64 * widths and "STG.E.128" in b, n
    for k in bwd.values():
        b = k.sass
        assert "UTMALDG" in b and b.count("ATOMS.ADD") >= 256 and "REDG.E.ADD.F32x4" in b and "ATOMS.CAST" not in b
    expanded_ac = {n: k.sass for n, k in {**fwd, **bwd}.items() if k.key in (KEY_STAGED | KEY_AC, KEY_BWD | KEY_STAGED | KEY_AC)}
    assert len(expanded_ac) == 2
    for n, b in expanded_ac.items():                             # the two instantiations the headline bench runs
        local = b.count(" STL") + b.count(" LDL")
        # forward: no spills.  Backward: sm_90 ptxas keeps one tile counter in local memory (one store + one load per tile of
        # 24 x 64 pixels, outside the plane loop); nothing more may spill.
        assert local == 0 if "fwd" in n else local <= 4, (n, local)
