"""ctypes binding of the C ABI in include/gmpi_mpi_render.h.

There is no CPU or PyTorch fallback: if the library is missing or fails to load this raises."""
import ctypes
import os

from ._build import LIB_PATH

GMPI_OK = 0
FLAG_RGBA_RANGE = 1
FLAG_ALPHA_RANGE = 2
FLAG_LAST_PLANE_OOB = 4
FLAG_PLANE_BEHIND_EYE = 8

OPT_ALIGN_CORNERS = 1
OPT_CHECK_LAST_PLANE = 2
OPT_COLOR_MINUS1_1 = 4
OPT_ZERO_GRAD = 8

PLAN_DIRECT, PLAN_STAGED = 1, 2
WHY = {1: "texture width is not a multiple of 4 (8 in fp16, 16 in uint8)", 2: "fewer than 120 tiles of 64x30 pixels",
       4: "more than 512 planes, or 2^31 planes over all MPIs", 8: "an MPI base pointer is not 16-byte aligned",
       16: "direct kernel forced by gmpi_debug_set_fwd_variant",
       # the backward's own (gmpi_mpi_render_bwd_plan_ex)
       32: "no saved transmittance", 64: "image width is not a multiple of 4",
       128: "a gradient or transmittance base pointer is not 16-byte aligned", 256: "2^31 or more pixel planes (V*N)"}

ABI_VERSION = 2

OPT_U8_ROUND_HALF_UP = 16
OPT_EARLY_STOP = 32
OPT_MPI_F16 = 64
OPT_MPI_U8 = 128


class RenderDesc(ctypes.Structure):
    """gmpi_render_desc of include/gmpi_mpi_render.h (field for field)."""
    _fields_ = [("struct_bytes", ctypes.c_uint32), ("options", ctypes.c_uint32),
                ("M", ctypes.c_int32), ("V", ctypes.c_int32), ("N", ctypes.c_int32), ("Ht", ctypes.c_int32), ("Wt", ctypes.c_int32),
                ("H", ctypes.c_int32), ("W", ctypes.c_int32), ("view_group", ctypes.c_int32),
                ("n_peers", ctypes.c_int32), ("frame_offset", ctypes.c_int32),
                ("depth_near", ctypes.c_float), ("depth_range", ctypes.c_float)] + \
               [(n, ctypes.c_void_p) for n in ("rgba", "rgb", "alpha", "bg_rgb", "view2mpi", "dhw", "ray_dir", "eye", "z_dir", "cam",
                                               "color", "depth", "transmittance", "peer_frames", "video_rgb", "video_depth",
                                               "g_color", "g_depth", "g_rgba", "g_rgb", "g_bg_rgb", "g_alpha", "flags", "stream")] + \
               [("early_stop", ctypes.c_float)]

# struct_bytes of a descriptor built against the header before early_stop was appended (GMPI_RENDER_DESC_V2_BYTES)
RENDER_DESC_V2_BYTES = RenderDesc.early_stop.offset


_vp, _i, _u32, _ll, _size, _desc = ctypes.c_void_p, ctypes.c_int, ctypes.c_uint32, ctypes.c_longlong, ctypes.c_size_t, \
    ctypes.POINTER(RenderDesc)
# {name: (restype, argtypes)} of every function the header declares, in its order
SIGNATURES = {
    "gmpi_abi_version": (_i, []),
    "gmpi_last_error": (ctypes.c_char_p, []),
    "gmpi_mpi_render_fwd_variant": (ctypes.c_char_p, [_i] * 5),
    "gmpi_mpi_render_fwd_plan": (_i, [_i] * 6 + [_vp, _vp]),
    "gmpi_mpi_render_fwd": (_i, [_vp] * 9 + [_i] * 7 + [_u32, _vp]),
    "gmpi_mpi_render_fwd_gather": (_i, [_vp] * 7 + [_i, _i, _vp] + [_i] * 7 + [_u32, _vp]),
    "gmpi_mpi_render_bwd": (_i, [_vp] * 9 + [_i] * 7 + [_u32, _vp]),
    "gmpi_mpi_render_fwd_train": (_i, [_vp] * 10 + [_i] * 7 + [_u32, _vp]),
    "gmpi_mpi_render_bwd_saved": (_i, [_vp] * 10 + [_i] * 7 + [_u32, _vp]),
    "gmpi_mpi_zero_async": (_i, [_vp, _size, _vp]),
    "gmpi_mpi_render_fwd_ex": (_i, [_desc]),
    "gmpi_mpi_render_fwd_plan_ex": (_i, [_desc, _vp]),
    "gmpi_mpi_render_bwd_plan_ex": (_i, [_desc, _vp]),
    "gmpi_mpi_render_bwd_ex": (_i, [_desc]),
    "gmpi_mpi_render_bwd_deterministic_scratch_bytes": (_ll, [_desc]),
    "gmpi_mpi_render_bwd_deterministic_ex": (_i, [_desc, _vp, _size]),
    "gmpi_mpi_occupancy_bytes": (_ll, [_desc]),
    "gmpi_mpi_build_occupancy": (_i, [_desc, _vp, _size]),
    "gmpi_mpi_render_fwd_skip_ex": (_i, [_desc, _vp, _size]),
    "gmpi_mpi_render_host_ex": (_i, [_desc, _i]),
    "gmpi_mpi_alpha_depth_fwd": (_i, [_vp, _ll, _ll, _vp, _vp, _vp] + [_i] * 4 + [_vp]),
    "gmpi_mpi_alpha_depth_bwd": (_i, [_vp, _ll, _ll, _vp, _vp, _vp, _vp, _ll, _ll] + [_i] * 4 + [_vp]),
    "gmpi_mpi_apply_shading_fwd": (_i, [_vp] * 3 + [_i] * 4 + [_vp]),
    "gmpi_mpi_apply_shading_bwd": (_i, [_vp] * 5 + [_i] * 4 + [_vp]),
    "gmpi_mpi_check_range": (_i, [_vp] + [_i] * 4 + [_vp, _vp]),
    "gmpi_mpi_check_range_f16": (_i, [_vp] + [_i] * 4 + [_vp, _vp]),
    "gmpi_mpi_render_fwd_host": (_i, [_vp] * 9 + [_i] * 7 + [_u32, _i]),
    "gmpi_mpi_release_host_cache": (_i, []),
    "gmpi_debug_plane_coords": (_i, [_vp] * 5 + [_i] * 6 + [_u32, _vp]),
    "gmpi_debug_plane_coords_packed": (_i, [_vp] * 5 + [_i] * 6 + [_u32, _vp]),
    "gmpi_debug_set_fwd_variant": (_i, [_i]),
    "gmpi_debug_set_fwd_stages": (_i, [_i]),
    "gmpi_debug_fwd_early_stop_stats": (_i, [_vp, _vp]),
    "gmpi_debug_fwd_skip_stats": (_i, [_vp, _vp]),
    "gmpi_debug_last_render_key": (_i, [_i, _vp]),
    "gmpi_debug_box_occupied": (_i, [_vp] + [_i] * 6),
    "gmpi_debug_u8_codes_host": (_i, [_vp]),
    "gmpi_debug_u8_codes": (_i, [_vp, _vp]),
    "gmpi_debug_fwd_ring_stages": (_i, [_i] * 6),
    "gmpi_debug_copy_plan": (_i, [_i, _vp, _i]),
    "gmpi_debug_tile_walk_ex": (_i, [_i] * 7 + [_vp, _i]),
    "gmpi_debug_cam_rays": (_i, [_vp, _vp, _i, _i, _i, _vp]),
    "gmpi_debug_tile_walk": (_i, [_i] * 5 + [_vp, _i]),
    "gmpi_debug_division": (_i, [_vp] * 4 + [_size, _vp]),
}
EXPORTS = sorted(SIGNATURES)


def make_desc(**kw) -> RenderDesc:
    """RenderDesc with struct_bytes set; tensors are passed as such (their data_ptr is taken), None -> NULL."""
    d = RenderDesc()
    d.struct_bytes = ctypes.sizeof(RenderDesc)
    for k, v in kw.items():
        if v is None:
            continue
        if hasattr(v, "data_ptr"):
            v = v.data_ptr()
        setattr(d, k, v)
    return d


_lib = None


class GmpiLibraryError(RuntimeError):
    pass


def load():
    global _lib
    if _lib is not None:
        return _lib
    path = os.environ.get("GMPI_LIB_PATH", LIB_PATH)     # override: A/B-testing kernel builds
    if not os.path.exists(path):
        raise GmpiLibraryError(
            f"{path} is missing: the CUDA (sm_90a) renderer is not built. Run "
            "`python -c 'import __graft_entry__ as g; g.build()'` (needs nvcc). There is no CPU fallback.")
    lib = ctypes.CDLL(path)
    for name, (restype, argtypes) in SIGNATURES.items():
        fn = getattr(lib, name)
        fn.restype, fn.argtypes = restype, argtypes
    if lib.gmpi_abi_version() != ABI_VERSION:
        raise GmpiLibraryError(f"ABI mismatch: library {lib.gmpi_abi_version()} != binding {ABI_VERSION}; rebuild")
    _lib = lib
    return lib


def check(rc: int):
    if rc != GMPI_OK:
        raise GmpiLibraryError(f"gmpi error {rc}: {load().gmpi_last_error().decode()}")


def deterministic_scratch_bytes(desc: RenderDesc) -> int:
    """Bytes of scratch gmpi_mpi_render_bwd_deterministic_ex needs for `desc` (raises on a bad descriptor)."""
    n = load().gmpi_mpi_render_bwd_deterministic_scratch_bytes(ctypes.byref(desc))
    if n < 0:
        check(-n)
    return n


def occupancy_bytes(desc: RenderDesc) -> int:
    """Bytes of the occupancy map of the MPI `desc` describes (gmpi_mpi_occupancy_bytes; raises on a bad descriptor)."""
    n = load().gmpi_mpi_occupancy_bytes(ctypes.byref(desc))
    if n < 0:
        check(-n)
    return n


def fwd_plan(desc: RenderDesc):
    """(plan, why) of the forward `desc` describes (gmpi_mpi_render_fwd_plan_ex): PLAN_STAGED or PLAN_DIRECT, and the WHY bits."""
    why = ctypes.c_uint32(0)
    plan = load().gmpi_mpi_render_fwd_plan_ex(ctypes.byref(desc), ctypes.byref(why))
    if plan < 0:
        check(-plan)
    return plan, why.value


def bwd_plan(desc: RenderDesc):
    """(plan, why) of the backward `desc` describes (gmpi_mpi_render_bwd_plan_ex): PLAN_STAGED (the box kernel) or PLAN_DIRECT, and
    the WHY bits; raises what the backward call would raise on the host."""
    why = ctypes.c_uint32(0)
    plan = load().gmpi_mpi_render_bwd_plan_ex(ctypes.byref(desc), ctypes.byref(why))
    if plan < 0:
        check(-plan)
    return plan, why.value


def reasons(why: int):
    """The WHY texts of the bits of `why`, in bit order."""
    return [t for b, t in WHY.items() if why & b]
