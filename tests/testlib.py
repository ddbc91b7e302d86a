"""Helpers the test modules share.  pytest does not collect this module; the tests import it as they import conftest.

  dev, lib                        the device of the GPU tests; the built library (module fixture of the CPU tests)
  KERNELS, set_kernel,            the forward-kernel switch: set both of its halves, force a kernel for a with block, or declare a
  forced_kernel, kernel_fixture   fixture that runs a test once per kernel
  misaligned, assert_bitwise      a copy at a given offset from a 16-byte boundary; dtype, shape and bytes equal
  early_stop_stats, skip_stats    the stage counters of the last staged forward
  case, synth_case, golden_case,  the case catalogue: every case of the GPU tests' edges as one record (geometry, expanded and
  CASES, FULL, on_device, pixels  factored MPI, upstream gradients); the forward tests' cases; the full-size shapes; a case's
                                  arrays on the device; the pixels a check compares
  shuffled_rays, corners_off,     the ray perturbations of the edge cases, and the views of a case in another order
  degenerate_rays, view_order
  forward_desc, render_fwd,       one gmpi_mpi_render_fwd_ex of a catalogue case, and the render of a native (fp16 / uint8) MPI
  native_vs_fp32                  beside the fp32 MPI it stands for, on the same kernel
  BIG_*, big_views                the shapes, views and declared device peaks of the buffers past 2^31 elements
  EXPECT, FACTORED_RGB_EXPECT     the parity bar against the CPU oracle, and the bar of a factored MPI's d rgb
  ORACLE_THREADS, to_np           the oracle's threads; a tensor as numpy
  upstream, oracle_forward,       the upstream gradients of a backward test; the oracle's forward and backward of a case; its
  oracle_backward, factored_refs, gradient split into a factored MPI's (d rgb, d alpha, d bg_rgb), and the check of a factored
  check_factored                  backward against it
and the helpers several modules read: the machine code of the built library, the staged forward's footprints,
oracle-side bounds and references, and the flag cases of tests/golden/flags_edges.npz."""
import contextlib
import ctypes
import dataclasses
import functools
import hashlib
import json
import os
import re
import subprocess
from typing import NamedTuple, Optional

import numpy as np
import pytest
import torch

from conftest import GOLDEN, MPI_CASES, load_golden, rel_err     # first: it puts the repository and oracle/ on sys.path
import mpi_oracle  # noqa: E402
import ml_gmpi_b200 as g  # noqa: E402
from ml_gmpi_b200 import _lib, synth  # noqa: E402


def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.fixture(scope="module")
def lib():
    g.build_library()
    return _lib.load()


# ------------------------------------------------------------------------------------------------------------------------------
# the kernel switch (process-wide: every render after set_kernel takes the forced kernel)
# ------------------------------------------------------------------------------------------------------------------------------
# name: (gmpi_debug_set_fwd_variant, gmpi_debug_set_fwd_stages) -- the kernel (automatic, direct, TMA-staged) and the staged
# forward's ring depth (0: the depth it picks itself; the factored forward's ring is always 3 deep)
KERNELS = {"auto": (0, 0), "direct": (1, 0), "staged": (2, 0), "staged2": (2, 2), "staged3": (2, 3)}


def set_kernel(name):
    """Forces the kernel and the ring depth of `name`, both."""
    variant, stages = KERNELS[name]
    lib = _lib.load()
    _lib.check(lib.gmpi_debug_set_fwd_variant(variant))
    _lib.check(lib.gmpi_debug_set_fwd_stages(stages))


@contextlib.contextmanager
def forced_kernel(name):
    """The kernel `name` inside the with block, the automatic choice after it, also when the block raises."""
    set_kernel(name)
    try:
        yield name
    finally:
        set_kernel("auto")


def kernel_fixture(*names):
    """A fixture that runs each test once per kernel name, forced as by forced_kernel; its value is the name.  The module attribute
    it is assigned to names it: `variant = kernel_fixture("direct", "staged2", "staged3")`."""
    @pytest.fixture(params=list(names))
    def fixture(request):
        with forced_kernel(request.param):
            yield request.param
    return fixture


# ------------------------------------------------------------------------------------------------------------------------------
# buffers, bits, counters
# ------------------------------------------------------------------------------------------------------------------------------
def misaligned(x, offset):
    """x's values in a buffer whose base is `offset` bytes (a multiple of x's element size) past a 16-byte boundary."""
    size = x.element_size()
    buf = torch.empty(x.numel() + 16 // size, dtype=x.dtype, device=x.device)
    start = (offset - buf.data_ptr()) % 16 // size
    y = buf[start:start + x.numel()].view(x.shape)
    y.copy_(x)
    assert y.data_ptr() % 16 == offset, (y.data_ptr() % 16, offset)
    return y


def assert_bitwise(a, b, what=None):
    """a and b have the same dtype, shape and bytes.  Each is a numpy array, a torch tensor or a number, or a list or tuple of them
    (then both have the same length and are compared element by element).  `what` names the case in the message."""
    if isinstance(a, (list, tuple)):
        assert isinstance(b, (list, tuple)) and len(a) == len(b), (what, "lengths differ")
        for i, (x, y) in enumerate(zip(a, b)):
            assert_bitwise(x, y, (what, i))
        return
    x, y = (t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else np.asarray(t) for t in (a, b))
    assert x.dtype == y.dtype and x.shape == y.shape, (what, x.dtype, x.shape, y.dtype, y.shape)
    if x.tobytes() != y.tobytes():
        with np.errstate(invalid="ignore"):
            diff = np.abs(x.astype(np.float64) - y.astype(np.float64))
        raise AssertionError((what, "max |a - b|", float(np.nanmax(diff, initial=0.0))))


def _stage_counts(fn):
    s, t = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
    _lib.check(fn(ctypes.byref(s), ctypes.byref(t)))
    return s.value, t.value


def early_stop_stats():
    """(stages stopped early, stages counted) of the last forward (gmpi_debug_fwd_early_stop_stats)."""
    return _stage_counts(_lib.load().gmpi_debug_fwd_early_stop_stats)


def skip_stats():
    """(stages skipped as empty, stages counted) of the last forward (gmpi_debug_fwd_skip_stats)."""
    return _stage_counts(_lib.load().gmpi_debug_fwd_skip_stats)


# ------------------------------------------------------------------------------------------------------------------------------
# the case catalogue: every case of the GPU tests' edges, as one record of numpy arrays, built once
# ------------------------------------------------------------------------------------------------------------------------------
# A record holds the geometry (view2mpi, dhw, ray_dir, eye, z_dir, ac: align_corners, view_group); an expanded MPI rgba with its own
# colour on every plane; a factored MPI (rgb, alpha, bg) over the same texture, whose alpha is rgba's; the upstream gradients of a
# backward (gc, and gd or None without a depth gradient).  Optional fields: factored (the forward tests render the factors: rgba is
# then their expanded stack), video (uint8 video frames), m11 (colour in [-1, 1]), visible (the background shows through: the
# alphas in front of the last plane are scaled down), ok ([V,H,W]: the pixels the checks compare; the others get no upstream
# gradient), and for the golden fixtures the reference's colour and depth.
GEOMETRY = ("dhw", "view2mpi", "ray_dir", "eye", "z_dir")      # in the order render_views takes them


def golden_case(name):
    """A golden fixture as a record: its inputs, the reference's colour and depth, its upstream gradients; the factored MPI is
    plane 0's colour, every plane's alpha and the last plane's colour."""
    gd = load_golden(name)
    rgba = gd["rgba"]
    return dict({k: gd[k] for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir", "color", "depth")}, ac=bool(gd["align_corners"]),
                rgb=rgba[:, 0, :3].copy(), alpha=rgba[:, :, 3:4].copy(), bg=rgba[:, -1, :3].copy(), gc=gd["g_color"], gd=gd.get("g_depth"))


def synth_case(*, n_planes, tex, img, n_mpi, views_per_mpi=1, seed, last_alpha_one=True, alpha="uniform", yaws=None, pitches=None,
               tex_hw=None, alpha_scale=None, plane=None, crop=None, rays=None, extra_mpis=0, ac=True, view_group=1, factored=False,
               video=False, depth_grad=True, m11=False, visible=False):
    """A record of synth.make_case's geometry (its first arguments, FULL's keys) and an MPI drawn as make_case draws it, U(0, 1) from
    a CPU generator seeded with `seed` (alpha: "uniform", or "equal_weight", synth.equal_weight_alpha), [n_mpi + extra_mpis, n_planes,
    4, *tex_hw] (tex_hw: (tex, tex)); alpha_scale scales the alphas in front of the last plane.  rgb and bg are drawn from seed + 1.
    plane: take plane `plane` of an n_planes table (then the MPI has one plane); crop: rows crop[0]:crop[1] of the image; rays: a
    function of the ray tensor (shuffled_rays, corners_off, degenerate_rays); extra_mpis: MPIs that no view looks at.  The upstream
    gradients are upstream(V, H, W, seed, depth_grad)."""
    geo = synth.make_case(n_planes=n_planes, tex=8, img=img, n_mpi=n_mpi, views_per_mpi=views_per_mpi, seed=seed, yaws=yaws,
                          pitches=pitches, rgba=False)
    dhw = geo.dhw if plane is None else geo.dhw[:, plane:plane + 1]
    M, N, tex_hw = n_mpi + extra_mpis, dhw.shape[1], tex_hw or (tex, tex)
    gen = torch.Generator().manual_seed(seed)
    rgba = torch.rand((M, N, 4) + tex_hw, generator=gen)
    if alpha == "equal_weight":
        rgba[:, :, 3] = synth.equal_weight_alpha((M, N) + tex_hw, gen)
    if alpha_scale is not None:
        rgba[:, :-1, 3] *= alpha_scale
    if last_alpha_one:
        rgba[:, -1, 3] = 1.0
    gen = torch.Generator().manual_seed(seed + 1)
    rgb, bg = torch.rand((M, 3) + tex_hw, generator=gen), torch.rand((M, 3) + tex_hw, generator=gen)
    alpha = rgba[:, :, 3:4].contiguous()
    if factored:      # one shared colour image, the last plane's own colour, per-plane alpha
        rgba = g.expand_factored(rgb, alpha, bg)
    ray = geo.ray_dir if crop is None else geo.ray_dir[:, :, crop[0]:crop[1]]
    ray = ray.contiguous() if rays is None else rays(ray)
    V, _, H, W = ray.shape
    gc, gd = upstream(V, H, W, seed, depth_grad)
    c = dict(rgba=rgba, rgb=rgb, alpha=alpha, bg=bg, view2mpi=geo.view2mpi, dhw=dhw[:1].expand(M, -1, -1), ray_dir=ray, eye=geo.eye,
             z_dir=geo.z_dir, gc=gc, gd=gd)
    c = {k: None if t is None else np.ascontiguousarray(t.numpy()) for k, t in c.items()}
    c.update(ac=ac, view_group=view_group, video=video, m11=m11, visible=visible)
    if factored:
        c["factored"] = True
    ok = np.isfinite(c["ray_dir"]).all(1) & (c["ray_dir"][:, 2] != 0)
    if not ok.all():
        c["ok"] = ok
        c["gc"] *= ok[:, None]
    return c


def shuffled_rays(ray):
    """The rays shuffled over the image (one permutation for every view): not a pinhole camera's, so no tile's corner rays bound
    its taps."""
    V, _, H, W = ray.shape
    perm = torch.randperm(H * W, generator=torch.Generator().manual_seed(0))
    return ray.reshape(V, 3, -1)[:, :, perm].reshape(V, 3, H, W).contiguous()


TILE_W = 64          # kTileW: the pixel columns of a tile of the staged kernels (csrc/mpi_fwd_staged.cuh)


def corners_off(ray):
    """The four corner rays of every TILE_W x FWD_TILE[0] tile of the staged forward pushed far off the planes, the interior rays
    kept."""
    ray = ray.clone()
    H, W = ray.shape[-2:]
    tw, th = TILE_W, mpi_oracle.FWD_TILE[0]
    for ty in range(0, H, th):
        for tx in range(0, W, tw):
            for cy in (ty, min(ty + th - 1, H - 1)):
                for cx in (tx, min(tx + tw - 1, W - 1)):
                    ray[:, 0, cy, cx] = 5.0
    return ray


def degenerate_rays(ray):
    """View 0's rays at (10, 10:14) parallel to the planes (ray_z == 0), and a NaN ray at (20, 20)."""
    ray = ray.clone()
    ray[0, 2, 10, 10:14] = 0.0
    ray[0, :, 20, 20] = float("nan")
    return ray


VIEW_ORDERS = {"sorted": [0, 1, 2, 3, 4, 5], "interleaved": [0, 2, 4, 1, 3, 5], "reversed": [5, 4, 3, 2, 1, 0]}


def view_order(c, order):
    """Case c with its views (rays, poses and upstream gradients) in the order VIEW_ORDERS[order] of six views."""
    perm = VIEW_ORDERS[order]
    return dict(c, **{k: None if c[k] is None else np.ascontiguousarray(c[k][perm]) for k in ("view2mpi", "ray_dir", "eye", "z_dir",
                                                                                                 "gc", "gd")})


# The full-size shapes (BASELINE.json's configs): synth.make_case arguments
C4_YAWS = np.linspace(0.5, -0.5, 120).astype(np.float32)[::8]
FULL = {
    "full_32x256": dict(n_planes=32, tex=256, img=256, n_mpi=8, seed=1234),
    "full_96x512": dict(n_planes=96, tex=512, img=512, n_mpi=2, seed=1234),
    "full_96x1024": dict(n_planes=96, tex=1024, img=1024, n_mpi=1, seed=1234),
    "c3": dict(n_planes=96, tex=1024, img=1024, n_mpi=1, seed=1234, last_alpha_one=True),
    "ffhq1024_batch4": dict(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=1234, last_alpha_one=True),   # bench.py's batch: 6.4 GB
    "c5": dict(n_planes=96, tex=512, img=512, n_mpi=4, seed=99, last_alpha_one=True),
    "four_views": dict(n_planes=48, tex=512, img=512, n_mpi=1, views_per_mpi=4, seed=21, last_alpha_one=True),
    "c4_video": dict(n_planes=96, tex=512, img=512, n_mpi=1, views_per_mpi=15, seed=1234, yaws=C4_YAWS, pitches=np.zeros(15, np.float32)),
}


def _bench(alpha):
    """bench.py's shape for one view: 96 planes, 1024^2, no opaque last plane, colour-only upstream gradient w.r.t. 2c - 1."""
    return synth_case(**FULL["full_96x1024"], last_alpha_one=False, alpha=alpha, depth_grad=False, m11=True)


def _views4(alpha):
    """One 48-plane 512^2 MPI seen from four views, colour and depth upstream gradients, alpha == 1 last plane."""
    return synth_case(**FULL["four_views"], alpha=alpha)


def _wide(wt, seed):
    """16 planes of a 512 x wt texture at 720^2 from three random poses: 1.4 texels per pixel across a tile (64 pixels), 0.7 down
    it.  wt = 1024: many (tile, plane) footprints need the widest box classes (85..88; 89..96, which the factored forward's 96-wide
    box could hold but which take the generic body), at origins where the fp16 box starts 4 texels further west and at every
    offset from the uint8 box's multiple of 16; wt = 1536: footprints wider than 96."""
    return synth_case(n_planes=16, tex=None, img=720, n_mpi=1, views_per_mpi=3, seed=seed, tex_hw=(512, wt), alpha_scale=0.1,
                      visible=True)


SYNTH = {
    "small": lambda: synth_case(n_planes=16, tex=64, img=96, n_mpi=2, views_per_mpi=2, seed=1),
    "view_group3": lambda: synth_case(n_planes=24, tex=96, img=128, n_mpi=1, views_per_mpi=3, seed=2, view_group=3),
    "factored": lambda: synth_case(n_planes=24, tex=96, img=128, n_mpi=2, views_per_mpi=2, seed=3, factored=True),
    "factored_view_group2": lambda: synth_case(n_planes=12, tex=64, img=96, n_mpi=1, views_per_mpi=2, seed=4, factored=True,
                                               view_group=2),
    "uint8": lambda: synth_case(n_planes=16, tex=64, img=96, n_mpi=2, views_per_mpi=2, seed=5, video=True),
    # the edges: one plane that is not opaque (plane 3 of an 8-plane table); N = kMaxPlanesStaged, whose back planes show through;
    # 100 x 136 pixels (partial tiles of the forward's 64 x 30 and the backward's 64 x 24) cut out of a pinhole image, a 72 x 116
    # texture (116 % 8 == 116 % 16 == 4), align_corners=False
    "N1": lambda: synth_case(n_planes=8, plane=3, tex=128, img=160, n_mpi=2, seed=41, last_alpha_one=False, visible=True),
    "N2": lambda: synth_case(n_planes=2, tex=128, img=160, n_mpi=2, seed=7),
    "N512": lambda: synth_case(n_planes=512, tex=96, img=128, n_mpi=2, seed=43, alpha_scale=0.02),
    "partial_acfalse_nonsquare": lambda: synth_case(n_planes=10, tex=None, img=136, n_mpi=2, views_per_mpi=2, seed=47, tex_hw=(72, 116),
                                                    alpha_scale=0.2, crop=(18, 118), ac=False, visible=True),
    "shuffled_rays": lambda: synth_case(n_planes=12, tex=96, img=200, n_mpi=1, views_per_mpi=2, seed=3, alpha_scale=0.2,
                                        rays=shuffled_rays, visible=True),
    "corners_off_the_planes": lambda: synth_case(n_planes=6, tex=64, img=128, n_mpi=1, views_per_mpi=2, seed=9, alpha_scale=0.4,
                                                 rays=corners_off, visible=True),
    "degenerate_rays": lambda: synth_case(n_planes=8, tex=64, img=64, n_mpi=1, seed=4, alpha_scale=0.3, rays=degenerate_rays,
                                          depth_grad=False, visible=True),
    # three MPIs of two views each and a fourth MPI that no view looks at, views in every order of VIEW_ORDERS
    "three_mpis": lambda: synth_case(n_planes=12, tex=256, img=256, n_mpi=3, views_per_mpi=2, seed=77, alpha_scale=0.15, extra_mpis=1,
                                     visible=True),
    **{f"three_mpis_{o}": (lambda o=o: view_order(case("three_mpis"), o)) for o in VIEW_ORDERS},
    "band_89_96": lambda: _wide(1024, 21),
    "wider_than_96": lambda: _wide(1536, 22),
    "bench_96x1024": lambda: _bench("uniform"),
    "views4_48x512": lambda: _views4("uniform"),
    # the operating points with every plane visible: U(0, 1) alpha hides the planes past ~25 from every bar
    "bench_96x1024_equal_weight": lambda: _bench("equal_weight"),
    "views4_48x512_equal_weight": lambda: _views4("equal_weight"),
    # the cases of the transmittance and factored suites' own tests
    "small_12x96": lambda: synth_case(n_planes=12, tex=96, img=128, n_mpi=2, views_per_mpi=2, seed=5, alpha_scale=0.18, visible=True),
    "staged_shape": lambda: synth_case(n_planes=12, tex=96, img=256, n_mpi=2, views_per_mpi=2, seed=6, alpha_scale=0.25),
    "bench_96x512_one_view": lambda: synth_case(n_planes=96, tex=512, img=512, n_mpi=1, seed=1234, alpha_scale=0.06),
    "view_group": lambda: synth_case(n_planes=16, tex=256, img=256, n_mpi=2, views_per_mpi=4, seed=8, alpha_scale=0.12, visible=True),
}


@functools.lru_cache(maxsize=None)
def case(name):
    return SYNTH[name]() if name in SYNTH else golden_case(name)


# the forward tests' cases (fp16, uint8, early stop)
CASES = MPI_CASES + ["c1_full_256", "small", "view_group3", "factored", "factored_view_group2", "uint8", "N1", "N2", "N512",
                     "partial_acfalse_nonsquare"]


def on_device(c, *keys):
    """The arrays `keys` of case c as tensors on the device (None stays None)."""
    return tuple(None if c[k] is None else torch.from_numpy(np.ascontiguousarray(c[k])).to(dev()) for k in keys)


def pixels(c, a):
    """a [V,C,H,W] at the pixels the checks compare: every pixel, or those of the case's mask ok, as [C, pixels]."""
    return a if c.get("ok") is None else a.transpose(1, 0, 2, 3)[:, c["ok"]]


# ------------------------------------------------------------------------------------------------------------------------------
# one forward through the descriptor, and the native-versus-fp32 harness of the fp16 and uint8 tests
# ------------------------------------------------------------------------------------------------------------------------------
_ELEMENT_OPTION = {torch.float32: 0, torch.float16: _lib.OPT_MPI_F16, torch.uint8: _lib.OPT_MPI_U8}


def forward_desc(c, mpi, tau=None, cam=None, u8_round=False, view_group=None, gather=False):
    """The descriptor of a forward of catalogue case c on the device MPI `mpi` ({"rgba": ...} or {"rgb", "alpha", "bg_rgb"}; its
    dtype sets the element option): the case's rays or the camera `cam`; colour and depth in [-1, 1], the uint8 video frames of a
    video case, or with `gather` the frames of a fused gather into one local buffer ("frames"); early stop at tau; the case's view
    group unless one is given.  Returns (descriptor, the tensors behind its pointers)."""
    d = dev()
    geo = dict(zip(GEOMETRY, on_device(c, *GEOMETRY)))
    ref = mpi["alpha"] if "alpha" in mpi else mpi["rgba"]
    V, _, H, W = c["ray_dir"].shape
    if gather:
        frames = torch.full((V, 4, H, W), float("nan"), device=d)
        out = dict(peer_frames=torch.tensor([frames.data_ptr()], dtype=torch.int64, device=d), n_peers=1, frame_offset=0)
    elif c.get("video"):
        out = dict(video_rgb=torch.empty((V, H, W, 3), dtype=torch.uint8, device=d),
                   video_depth=torch.empty((V, H, W, 1), dtype=torch.uint8, device=d), depth_near=0.9, depth_range=np.float32(0.3).item())
    else:
        out = dict(color=torch.empty((V, 3, H, W), device=d), depth=torch.empty((V, 1, H, W), device=d))
    rays = dict(cam=cam) if cam is not None else {k: geo[k] for k in ("ray_dir", "eye", "z_dir")}
    opts = (_lib.OPT_ALIGN_CORNERS if c["ac"] else 0) | _lib.OPT_COLOR_MINUS1_1 | (_lib.OPT_U8_ROUND_HALF_UP if u8_round else 0) \
        | (_lib.OPT_EARLY_STOP if tau is not None else 0) | _ELEMENT_OPTION[ref.dtype]
    keep = dict(view2mpi=geo["view2mpi"], dhw=geo["dhw"], flags=torch.zeros(1, dtype=torch.int32, device=d), **rays, **out, **mpi)
    desc = _lib.make_desc(options=opts, M=ref.shape[0], V=V, N=ref.shape[1], Ht=ref.shape[-2], Wt=ref.shape[-1], H=H, W=W,
                          view_group=c.get("view_group", 1) if view_group is None else view_group, early_stop=tau, **keep)
    return desc, dict(keep, frames=frames) if gather else keep


def render_fwd(c, mpi, **kw):
    """(outputs..., flags) of one gmpi_mpi_render_fwd_ex of forward_desc(c, mpi, **kw), as numpy."""
    desc, keep = forward_desc(c, mpi, **kw)
    _lib.check(_lib.load().gmpi_mpi_render_fwd_ex(ctypes.byref(desc)))
    torch.cuda.synchronize()
    names = ("frames",) if "frames" in keep else ("video_rgb", "video_depth") if "video_rgb" in keep else ("color", "depth")
    return tuple(keep[n].cpu().numpy() for n in names + ("flags",))


def native_vs_fp32(c, native, fp32, variant, **kw):
    """render_fwd of the native MPI `native` (fp16 or uint8) and of the fp32 MPI `fp32` it stands for, both on the kernel the native
    call gets under the forced kernel `variant`: where the plan query sends the native MPI to the direct kernel, the fp32 MPI renders
    there too.  Returns (native outputs, fp32 outputs, whether the native call fell back to the direct kernel)."""
    h = render_fwd(c, native, **kw)
    desc, _ = forward_desc(c, native, **{k: v for k, v in kw.items() if k != "gather"})
    fell_back = variant != "direct" and _lib.fwd_plan(desc)[0] == _lib.PLAN_DIRECT
    if fell_back:
        set_kernel("direct")
    try:
        f = render_fwd(c, fp32, **kw)
    finally:
        set_kernel(variant)
    return h, f, fell_back


# ------------------------------------------------------------------------------------------------------------------------------
# the staged forward's footprints and the cases at its widest box classes
# ------------------------------------------------------------------------------------------------------------------------------
def footprints(c):
    """mpi_oracle.footprints of case c's staged forward (the producer's box of every (view, tile, plane) stage)."""
    M, N, _, Ht, Wt = c["rgba"].shape
    return mpi_oracle.footprints(c["view2mpi"], c["dhw"], c["ray_dir"], c["eye"], Ht, Wt, c["ac"])


def limit_footprints(c, lo, hi):
    """(tile, plane) stages whose fp32 box lies under the tile with rows that fit a stage (mode 0, or mode 2 only for a width need
    above kMaxBW = 88) with a width need in [lo, hi] and an origin 4 texels past a multiple of 8."""
    f = footprints(c)
    fits = (f["mode"] != 1) & (-(-f["need_h"] // 4) * 4 <= mpi_oracle.FWD_TILE[1])
    return int((fits & (f["need_w"] >= lo) & (f["need_w"] <= hi) & (f["bx0"] % 8 == 4)).sum())


@functools.lru_cache(maxsize=None)
def headline_case():
    """One view of the headline MPI, 96 x 1024^2, with equal-weight alpha (synth.equal_weight_alpha): every plane, the back ones
    with the widest boxes included, reaches the render, so a back-plane tap the native kernel staged or converted wrongly changes
    the bits of the output (with U(0, 1) alpha it would be absorbed by the rounding of the accumulator)."""
    cs = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=1, seed=1234, alpha="equal_weight")
    return dict(rgba=cs.rgba.numpy(), view2mpi=cs.view2mpi.numpy(), dhw=cs.dhw.numpy(), ray_dir=cs.ray_dir.numpy(),
                eye=cs.eye.numpy(), z_dir=cs.z_dir.numpy(), ac=True)


# ------------------------------------------------------------------------------------------------------------------------------
# buffers past 2^31 elements (tests/test_gpu_large_offsets.py runs them; tests/test_large_offsets.py checks their arithmetic)
# ------------------------------------------------------------------------------------------------------------------------------
BIG_N, BIG_R = 96, 1024
BIG_IMG = BIG_R * BIG_R
BIG_MPI = BIG_N * 4 * BIG_IMG       # elements of one expanded 96 x 1024^2 MPI
BIG_SLABS = BIG_N * BIG_IMG         # elements of one factored alpha, or of one view's saved transmittance
BIG_M = 6                           # expanded MPIs in the far buffer: MPI 5 starts at element 2,013,265,920
BIG_M_FACTORED = 22                 # factored alphas, and views of saved transmittance: the last starts at 2,113,929,216
BIG_V_COLOR, BIG_V_GATHER = 684, 513        # colour / video frames, fused-gather frames of 1024^2 pixels
SMALL_MPI = dict(N=8, R=256)        # the MPI of the output tests
BIG_SLACK = 1 << 28                 # views, rays, outputs of a few views, flags and occupancy maps: under 256 MiB in every test

# test key: the device bytes its buffers hold at its peak, from the shapes above (BIG_SLACK on top)
BIG_PEAK_BYTES = {
    # far buffer, the fp32 MPI uploaded, the native MPI and its fp32 conversion
    "expanded_forward-fp32": BIG_M * BIG_MPI * 4 + BIG_MPI * 4,
    "expanded_forward-fp16": BIG_M * BIG_MPI * 2 + BIG_MPI * 4 + BIG_MPI * 2 + BIG_MPI * 4,
    "expanded_forward-uint8": BIG_M * BIG_MPI + BIG_MPI * 4 + BIG_MPI + BIG_MPI * 4,
    "wrong_inputs": BIG_M * BIG_MPI * 4 + 2 * BIG_MPI * 4,
    "skipping": BIG_M * BIG_MPI * 4 + BIG_MPI * 4,
    # rgba and g_rgba, the upload, two views' transmittance
    "expanded_backward": 2 * BIG_M * BIG_MPI * 4 + BIG_MPI * 4 + 2 * BIG_SLABS * 4,
    # alpha and g_alpha, rgb / bg_rgb and their gradients, the one MPI's factors, two views' transmittance
    "factored": 2 * BIG_M_FACTORED * BIG_SLABS * 4 + 4 * BIG_M_FACTORED * 3 * BIG_IMG * 4 + (BIG_SLABS + 6 * BIG_IMG) * 4
                + 2 * BIG_SLABS * 4,
    # transmittance, rgba and g_rgba, 8 B of deterministic scratch per gradient element, rays / colour / upstream of 22 views
    "saved_transmittance": BIG_M_FACTORED * BIG_SLABS * 4 + 2 * BIG_MPI * 4 + BIG_MPI * 8 + 4 * BIG_M_FACTORED * 4 * BIG_IMG * 4,
    # the frames, and in front of those past 2^31 elements 2^31 sentinels (where a signed 32-bit offset would wrap to)
    "outputs-color": (BIG_V_COLOR * 4 * BIG_IMG + (1 << 31)) * 4,
    "outputs-video": BIG_V_COLOR * 4 * BIG_IMG + (1 << 31),
    "outputs-gather": (BIG_V_GATHER * 4 * BIG_IMG + (1 << 31)) * 4,
    "range_check-fp32-vector": BIG_M * BIG_MPI * 4,
    "range_check-fp32-scalar": BIG_M * BIG_N * 4 * 1023 * 1023 * 4,
    "range_check-fp16-vector": BIG_M * BIG_MPI * 2,
    "range_check-fp16-scalar": BIG_M * BIG_N * 4 * 1023 * 1023 * 2,
    # the uint8 MPI on the device, and the host entry point's two staging slots (the library's own cudaMalloc: this is what the
    # test needs free, but torch's peak, which the budget fixture checks, does not see them)
    "host_entry_point": 3 * BIG_MPI,
    # the fp32 batch of four and the three temporaries of its equal-weight alpha (synth.equal_weight_alpha); the later steps (the
    # factored form, the fp16 and uint8 copies and their conversions) hold less
    "batch_of_four": 4 * BIG_MPI * 4 + 3 * 4 * BIG_SLABS * 4,
}


@functools.lru_cache(maxsize=None)
def big_views():
    """The two views of tests/test_gpu_large_offsets.py, both of MPI 0 (the caller moves them): view 0 is headline_case's pinhole
    view, whose stages take the staged forward's fast body at every box class; view 1 holds the same rays shuffled over the image,
    so no tile's corner rays bound its taps and every stage takes the generic body.  Geometry only: headline_case has the MPI."""
    cs = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=1, seed=1234, rgba=False)
    perm = torch.randperm(1024 * 1024, generator=torch.Generator().manual_seed(7))
    shuffled = cs.ray_dir.reshape(1, 3, -1)[:, :, perm].reshape(cs.ray_dir.shape)
    two = lambda t: torch.cat([t, t]).numpy()
    return dict(view2mpi=np.zeros(2, np.int32), dhw=cs.dhw.numpy(), ray_dir=torch.cat([cs.ray_dir, shuffled]).numpy(),
                eye=two(cs.eye), z_dir=two(cs.z_dir), ac=True)


def assert_class_88_behind_plane_25(c):
    cls = footprints(c)["cls"]
    assert (cls[..., 25:] == 88).any() and all((cls == k).any() for k in range(56, 96, 8))


# ------------------------------------------------------------------------------------------------------------------------------
# the CPU oracle (oracle/mpi_oracle.py): the parity bar, upstream gradients, the oracle's forward and backward of a case
# ------------------------------------------------------------------------------------------------------------------------------
# The parity bar: max |ours - oracle| / max |oracle| of colour, depth and d rgba.  The texel coordinates are bit-exact with the
# oracle's; the rest differs from it by fp32 summation order and FMA contraction, and by T <- T - w * 1 instead of
# T * (1 - a + 1e-10) (~1 ulp of T per plane): a few 1e-6.
EXPECT = 2e-5
# d rgb of a factored MPI sums the gradients of the N - 1 planes that share the colour image, so it sums their rounding errors too
# (fixed point in the kernels, fp32 in the oracle): twice the per-plane bar.
FACTORED_RGB_EXPECT = 2 * EXPECT
# The oracle's pthreads.  Its forward is the same on any number of them; the order of its backward's atomic float adds, hence
# the last ulp of the gradient, is not.
ORACLE_THREADS = max(1, min(64, os.cpu_count() or 8))


def to_np(t):
    """t as numpy: a tensor detached and copied to the CPU; an array, or None, as it is."""
    return t.detach().cpu().numpy() if isinstance(t, torch.Tensor) else t


def upstream(V, H, W, seed, depth=True, device=None):
    """(g_color [V,3,H,W], g_depth [V,1,H,W], or None without depth) of a backward test: randn, colour then depth, from a CPU
    generator seeded with `seed`, on `device` (the CPU if None)."""
    gen = torch.Generator().manual_seed(seed)
    gc = torch.randn((V, 3, H, W), generator=gen).to(device)
    return gc, torch.randn((V, 1, H, W), generator=gen).to(device) if depth else None


def _oracle_inputs(case, rgba, ray_dir):
    get = (lambda k: case[k]) if isinstance(case, dict) else (lambda k: getattr(case, k))
    given = dict(rgba=rgba, ray_dir=ray_dir)
    return [to_np(get(k) if given.get(k) is None else given[k]) for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")]


def oracle_forward(case, rgba=None, ray_dir=None, align_corners=True, check_last_plane=False):
    """mpi_oracle.forward of a case -> (colour, depth, flags).  The case is a dict or an object (synth.Case) with the fields rgba,
    view2mpi, dhw, ray_dir, eye and z_dir, as numpy arrays or tensors; rgba and ray_dir, when given, replace the case's."""
    return mpi_oracle.forward(*_oracle_inputs(case, rgba, ray_dir), align_corners=align_corners, check_last_plane=check_last_plane,
                              nthreads=ORACLE_THREADS)


def oracle_backward(case, g_color, g_depth=None, rgba=None, ray_dir=None, align_corners=True, minus1_1=False):
    """mpi_oracle.backward of a case (as oracle_forward takes it) under the upstream gradients -> d rgba.  minus1_1: g_color is the
    gradient of the colour in [-1, 1], 2 c - 1, whose gradient with respect to c is 2 g_color."""
    gc = to_np(g_color)
    return mpi_oracle.backward(*_oracle_inputs(case, rgba, ray_dir), 2.0 * gc if minus1_1 else gc, to_np(g_depth),
                               align_corners=align_corners, nthreads=ORACLE_THREADS)


def factored_refs(ref):
    """The oracle's expanded gradient -> (d rgb, d alpha, d bg_rgb) of a factored MPI with a background plane: d rgb is the sum, in
    float64, over the planes that share the colour image."""
    return ref[:, :-1, :3].astype(np.float64).sum(1), ref[:, :, 3:4], ref[:, -1, :3]


def check_factored(ours, ref):
    """ours = (d rgb, d alpha, d bg_rgb) against factored_refs(ref): d rgb within FACTORED_RGB_EXPECT, the others within EXPECT."""
    e = [rel_err(o, r) for o, r in zip(ours, factored_refs(ref))]
    assert e[0] <= FACTORED_RGB_EXPECT and e[1] <= EXPECT and e[2] <= EXPECT, e


# ------------------------------------------------------------------------------------------------------------------------------
# references and bounds
# ------------------------------------------------------------------------------------------------------------------------------
def max_plane_depth(gd):
    """[V,1,H,W]: the largest |z-depth| of a pixel over the planes, (d - e_z) / r_z * (r . z_dir) (mpi.py:74-76,149-151)."""
    ray, eye, z = gd["ray_dir"].astype(np.float64), gd["eye"].astype(np.float64), gd["z_dir"].astype(np.float64)
    d = gd["dhw"][gd["view2mpi"], :, 0].astype(np.float64)                      # [V,N]
    zlen = np.einsum("vchw,vc->vhw", ray, z)
    t = (d[:, :, None, None] - eye[:, 2, None, None, None]) / ray[:, None, 2]    # [V,N,H,W]
    return np.max(np.abs(t * zlen[:, None]), axis=1, keepdims=True)


def video_reference(color_m11, depth, near, far):
    """gmpi/eval/vis/render_video.py:118-126, verbatim arithmetic on numpy float32 arrays."""
    img = color_m11.permute(0, 2, 3, 1).cpu().numpy()
    img = (img + 1) / 2.0
    img = (img * 255).astype(np.uint8)
    depth_map = depth.permute(0, 2, 3, 1).cpu().numpy()
    depth_map = (depth_map - near) / (far - near)
    depth_map = np.clip(depth_map, 0, 1)
    depth_map = (depth_map * 255).astype(np.uint8)
    return img, depth_map


ALPHAS = ["uniform", "equal_weight"]


def each_alpha(argnames, sets, indirect=()):
    """parametrize(argnames + ",alpha") over sets x ALPHAS.  The U(0, 1) sets keep the ids they had before the equal-weight input
    was added; the equal-weight ones end in "-equal_weight"."""
    params = []
    for alpha in ALPHAS:
        for vals in sets:
            vals = vals if isinstance(vals, tuple) else (vals,)
            ident = "-".join(str(v) for v in vals) + ("" if alpha == "uniform" else "-" + alpha)
            params.append(pytest.param(*vals, alpha, id=ident))
    return pytest.mark.parametrize(argnames + ",alpha", params, indirect=list(indirect))


def reference_signatures():
    with open(os.path.join(GOLDEN, "reference_signatures.json")) as f:
        return json.load(f)


# The flag word each verdict of the reference implies (oracle/make_golden_flags.py): the forward's with the last-plane check.  The
# forward never sets the range bits; without the last-plane check it never sets LAST_PLANE_OOB.
FORWARD_FLAGS = {"ok": 0, "alpha": 0, "behind-eye": mpi_oracle.FLAG_PLANE_BEHIND_EYE, "out-of-plane": mpi_oracle.FLAG_LAST_PLANE_OOB}


def load_flag_cases():
    """[(name, verdict, case)] of tests/golden/flags_edges.npz; a case has rgba, dhw, view2mpi, ray_dir, eye, z_dir, align_corners."""
    z = load_golden("flags_edges")
    out = []
    for name, verdict in zip(z["names"].tolist(), z["verdicts"].tolist()):
        c = {k: z["pool_%d" % int(z[f"{name}__{k}"])] for k in ("dhw", "view2mpi", "ray_dir", "eye", "z_dir", "align_corners")}
        r = z[f"{name}__rgba"]
        c["rgba"] = np.random.default_rng(int(r[0])).random(tuple(z[f"{name}__rgba_shape"].tolist()), dtype=np.float32)
        if len(r) > 1:
            c["rgba"][tuple(int(i) for i in r[1:])] = z[f"{name}__rgba_value"]
        out.append((name, verdict, c))
    return out


FLAG_CASES = load_flag_cases()


# ------------------------------------------------------------------------------------------------------------------------------
# gradients through the wrappers (tests of the staged backward's box)
# ------------------------------------------------------------------------------------------------------------------------------
def expanded_grad(rgba, case, gc, gd, ray=None):
    """d rgba of sum(colour * gc) (+ sum(depth * gd)) through render_views, as numpy."""
    x = rgba.clone().requires_grad_(True)
    color, depth = g.render_views(x, case.dhw, case.view2mpi, case.ray_dir if ray is None else ray, case.eye, case.z_dir)
    loss = (color * gc).sum()
    if gd is not None:
        loss = loss + (depth * gd).sum()
    loss.backward()
    return x.grad.cpu().numpy()


def factored_grads(rgb, alpha, bg, case, gc, gd, ray=None):
    """(d rgb, d alpha, d bg_rgb) of the same loss through render_views_factored, as numpy."""
    r, a, b = (t.clone().requires_grad_(True) for t in (rgb, alpha, bg))
    color, depth = g.render_views_factored(r, a, case.dhw, case.view2mpi, case.ray_dir if ray is None else ray, case.eye, case.z_dir,
                                           bg_rgb=b)
    loss = (color * gc).sum()
    if gd is not None:
        loss = loss + (depth * gd).sum()
    loss.backward()
    return r.grad.cpu().numpy(), a.grad.cpu().numpy(), b.grad.cpu().numpy()


def one_tile_per_mpi_case(d):
    """Two MPIs, one near-frontal view each, of ONE 64 x 24 backward tile (rows 20..43 of a 64^2 pinhole image): every
    (tile, plane) takes the box, and every texel of g_rgba receives exactly one flush per plane, so the result does not
    depend on the order of fp32 atomics."""
    case = synth.make_case(n_planes=6, tex=64, img=64, n_mpi=2, seed=13, device=d, last_alpha_one=True,
                           yaws=[0.05, -0.08], pitches=[0.02, -0.03])
    return dataclasses.replace(case, ray_dir=case.ray_dir[:, :, 20:44].contiguous())


# ------------------------------------------------------------------------------------------------------------------------------
# the machine code of a built library
# ------------------------------------------------------------------------------------------------------------------------------
# The render-kernel key bits (kKey*, csrc/mpi_kernel_keys.cuh)
KEY_AC, KEY_FAC, KEY_EMIT, KEY_ES, KEY_F16, KEY_STAGED, KEY_BWD, KEY_DET, KEY_SKIP, KEY_U8 = 1, 2, 4, 8, 16, 32, 64, 128, 256, 512


class Kernel(NamedTuple):
    template: str           # the C++ name: a kernel template, or a plain or extern "C" kernel
    key: Optional[int]      # the render kernel's key (template<uint32_t K>), None for other kernels
    sass: str
    regs: int
    stack: int
    local: int

    def digest(self):
        """sha256 of the SASS instructions (addresses and encodings included, no names or comments)"""
        lines = [l.strip() for l in self.sass.split("\n") if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
        return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def library_kernels(path=None):
    """{mangled name: Kernel} of a built library (cuobjdump -sass and -res-usage).  Kernels of namespace gmpi are
    _ZN4gmpi<length><name>..., and a uint32_t template argument K mangles as ILj<K>E."""
    path = path or g._build.LIB_PATH
    run = lambda flag: subprocess.run(["cuobjdump", flag, path], capture_output=True, text=True, check=True).stdout
    usage = {m[1]: (int(m[2]), int(m[3]), int(m[4]))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", run("-res-usage"))}
    out = {}
    for f in re.split(r"\n\s*Function : ", run("-sass"))[1:]:
        name, body = f.split("\n", 1)
        name = name.strip()
        template, key = name, None
        m = re.match(r"_ZN4gmpi(\d+)", name)
        if m:
            end = m.end() + int(m[1])
            template = name[m.end():end]
            k = re.match(r"ILj(\d+)EE", name[end:])
            key = int(k[1]) if k else None
        out[name] = Kernel(template, key, body, *usage[name])
    return out


def render_kernels(kernels, template, has=0, lacks=0):
    """{name: Kernel} of the instantiations of `template` whose key has every bit of `has` and none of `lacks`"""
    return {n: k for n, k in kernels.items() if k.template == template and k.key & has == has and not k.key & lacks}
