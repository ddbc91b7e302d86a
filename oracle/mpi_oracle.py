"""ctypes/numpy front-end of the CPU oracle (oracle/mpi_oracle.c).

TEST INFRASTRUCTURE ONLY -- see the header of mpi_oracle.c.  Imported by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs, never by the
product package.
"""
import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "libgmpi_oracle.so")
_lib = None

FLAG_RGBA_RANGE = 1
FLAG_ALPHA_RANGE = 2
FLAG_LAST_PLANE_OOB = 4
FLAG_PLANE_BEHIND_EYE = 8


def build(force: bool = False) -> str:
    src = os.path.join(_HERE, "mpi_oracle.c")
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(src):
        subprocess.run(["make", "-C", _HERE, "-B" if force else "-s", "libgmpi_oracle.so"], check=True,
                       stdout=subprocess.DEVNULL)
    return _SO


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(_SO):
            build()
        _lib = ctypes.CDLL(_SO)
        fp = ctypes.POINTER(ctypes.c_float)
        ip = ctypes.POINTER(ctypes.c_int32)
        i = ctypes.c_int
        _lib.gmpi_oracle_forward_mt.restype = ctypes.c_uint32
        _lib.gmpi_oracle_forward_mt.argtypes = [fp, ip, fp, fp, fp, fp, fp, fp] + [i] * 10
        _lib.gmpi_oracle_forward_over.restype = None
        _lib.gmpi_oracle_forward_over.argtypes = [fp, ip, fp, fp, fp, fp, fp, fp] + [i] * 8
        _lib.gmpi_oracle_backward_mt.restype = None
        _lib.gmpi_oracle_backward_mt.argtypes = [fp, ip, fp, fp, fp, fp, fp, fp, fp] + [i] * 9
        _lib.gmpi_oracle_coords.restype = None
        _lib.gmpi_oracle_coords.argtypes = [ip, fp, fp, fp, fp] + [i] * 7
        _lib.gmpi_oracle_check_range.restype = ctypes.c_uint32
        _lib.gmpi_oracle_check_range.argtypes = [fp, ctypes.c_size_t, i, i]
    return _lib


def _f(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(ctypes.POINTER(ctypes.c_float))


def _i(a):
    a = np.ascontiguousarray(a, dtype=np.int32)
    return a, a.ctypes.data_as(ctypes.POINTER(ctypes.c_int32))


def _shapes(rgba, ray_dir):
    M, N, C, Ht, Wt = rgba.shape
    V, three, H, W = ray_dir.shape
    assert C == 4 and three == 3
    return M, N, Ht, Wt, V, H, W


def forward(rgba, view2mpi, dhw, ray_dir, eye, z_dir, align_corners=True, check_last_plane=False,
            nthreads=1):
    """-> (color [V,3,H,W], depth [V,1,H,W], flags)"""
    M, N, Ht, Wt, V, H, W = _shapes(rgba, ray_dir)
    rgba, p_rgba = _f(rgba); v2m, p_v2m = _i(view2mpi); dhw, p_dhw = _f(dhw)
    ray_dir, p_ray = _f(ray_dir); eye, p_eye = _f(eye); z_dir, p_z = _f(z_dir)
    color = np.empty((V, 3, H, W), np.float32); depth = np.empty((V, 1, H, W), np.float32)
    flags = lib().gmpi_oracle_forward_mt(
        p_rgba, p_v2m, p_dhw, p_ray, p_eye, p_z,
        color.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        depth.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        M, V, N, Ht, Wt, H, W, int(bool(align_corners)), int(bool(check_last_plane)), int(nthreads))
    return color, depth, int(flags)


def forward_over(rgba, view2mpi, dhw, ray_dir, eye, z_dir, align_corners=True):
    M, N, Ht, Wt, V, H, W = _shapes(rgba, ray_dir)
    rgba, p_rgba = _f(rgba); v2m, p_v2m = _i(view2mpi); dhw, p_dhw = _f(dhw)
    ray_dir, p_ray = _f(ray_dir); eye, p_eye = _f(eye); z_dir, p_z = _f(z_dir)
    color = np.empty((V, 3, H, W), np.float32); depth = np.empty((V, 1, H, W), np.float32)
    lib().gmpi_oracle_forward_over(
        p_rgba, p_v2m, p_dhw, p_ray, p_eye, p_z,
        color.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        depth.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        M, V, N, Ht, Wt, H, W, int(bool(align_corners)))
    return color, depth


def backward(rgba, view2mpi, dhw, ray_dir, eye, z_dir, g_color, g_depth=None, align_corners=True, nthreads=1):
    """-> g_rgba [M,N,4,Ht,Wt].  nthreads > 1 splits each view's rows over pthreads (atomic float adds: the summation
    order, hence the last ulp, then varies from run to run; nthreads == 1 is the sequential reference sum)."""
    M, N, Ht, Wt, V, H, W = _shapes(rgba, ray_dir)
    rgba, p_rgba = _f(rgba); v2m, p_v2m = _i(view2mpi); dhw, p_dhw = _f(dhw)
    ray_dir, p_ray = _f(ray_dir); eye, p_eye = _f(eye); z_dir, p_z = _f(z_dir)
    g_color, p_gc = _f(g_color)
    if g_depth is None:
        p_gd = ctypes.POINTER(ctypes.c_float)()
    else:
        g_depth, p_gd = _f(g_depth)
    g_rgba = np.zeros((M, N, 4, Ht, Wt), np.float32)
    lib().gmpi_oracle_backward_mt(
        p_rgba, p_v2m, p_dhw, p_ray, p_eye, p_z, p_gc, p_gd,
        g_rgba.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
        M, V, N, Ht, Wt, H, W, int(bool(align_corners)), int(nthreads))
    return g_rgba


def coords(view2mpi, dhw, ray_dir, eye, Ht, Wt, align_corners=True):
    """-> texel coordinates [V,N,2,H,W] (ix, iy), the bit-exact stage."""
    V, _, H, W = ray_dir.shape
    N = dhw.shape[1]
    v2m, p_v2m = _i(view2mpi); dhw, p_dhw = _f(dhw)
    ray_dir, p_ray = _f(ray_dir); eye, p_eye = _f(eye)
    out = np.empty((V, N, 2, H, W), np.float32)
    lib().gmpi_oracle_coords(p_v2m, p_dhw, p_ray, p_eye,
                             out.ctypes.data_as(ctypes.POINTER(ctypes.c_float)),
                             V, N, Ht, Wt, H, W, int(bool(align_corners)))
    return out


FWD_TILE = (30, 44)    # staged forward: tile rows kTileH, box rows kMaxBH (csrc/mpi_fwd_staged.cuh)
BWD_TILE = (24, 36)    # box backward: kBwdTileH, kBwdMaxBH (csrc/mpi_bwd_box.cuh)


def footprints(view2mpi, dhw, ray_dir, eye, Ht, Wt, align_corners=True, tile=FWD_TILE, wide=False):
    """The staged producer's box of every (view, tile, plane) stage (staged_producer, csrc/mpi_fwd_staged.cuh), computed as it
    does from coords() of each 64 x tile[0] pixel tile's four corner pixels (clamped into the image).  -> dict of int64 arrays
    [V, tiles_y, tiles_x, N]: bx0 (box origin, a multiple of 4), need_w, need_h, mode (0 staged, 1 nothing under the tile, 2 the
    generic body) and cls (the box width of the class: 56..88 in steps of 8, or 64 / 96 in the factored forward's wide ring;
    0 where mode != 0).  tile: (tile rows, box rows) of the forward (FWD_TILE) or the backward (BWD_TILE)."""
    tile_h, max_bh = tile
    V, _, H, W = ray_dir.shape
    px, py = np.arange(0, W, 64), np.arange(0, H, tile_h)
    xs = np.stack([px, np.minimum(px + 63, W - 1)], -1).reshape(-1)
    ys = np.stack([py, np.minimum(py + tile_h - 1, H - 1)], -1).reshape(-1)
    corners = np.ascontiguousarray(np.asarray(ray_dir)[:, :, ys][:, :, :, xs])
    c = coords(view2mpi, dhw, corners, eye, Ht, Wt, align_corners)             # [V, N, 2, 2 tiles_y, 2 tiles_x]
    N = c.shape[1]
    c = c.reshape(V, N, 2, len(py), 2, len(px), 2).transpose(0, 3, 5, 1, 2, 4, 6).reshape(V, len(py), len(px), N, 2, 4)
    ok = np.abs(c) < 1e9                                                         # False for inf and NaN
    finite = ok.all(axis=(-2, -1))
    f = np.floor(np.where(ok, c, 0)).astype(np.int64)
    xmin, xmax, ymin, ymax = f[..., 0, :].min(-1), f[..., 0, :].max(-1), f[..., 1, :].min(-1), f[..., 1, :].max(-1)
    bx0, by0 = (xmin - 1) // 4 * 4, ymin - 1
    need_w, need_h = xmax - bx0 + 3, ymax - ymin + 4
    mode = np.where(~finite | (need_w > 88) | (-(-need_h // 4) * 4 > max_bh), 2,
                    np.where((bx0 > Wt - 1) | (bx0 + need_w - 1 < 0) | (by0 > Ht - 1) | (by0 + need_h - 1 < 0), 1, 0))
    cls = np.where(need_w <= 64, 64, 96) if wide else 56 + 8 * np.maximum(0, -(-(need_w - 56) // 8))
    return dict(bx0=bx0, need_w=need_w, need_h=need_h, mode=mode, cls=np.where(mode == 0, cls, 0))


def check_range(rgba):
    M, N, _, Ht, Wt = rgba.shape
    rgba, p = _f(rgba)
    return int(lib().gmpi_oracle_check_range(p, M * N, Ht, Wt))
