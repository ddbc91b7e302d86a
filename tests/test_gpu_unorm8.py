"""GPU tests of 8-bit RGBA MPIs (GMPI_MPI_U8) on an H100: pytest -m gpu.

Code b of a uint8 MPI stands for b / 255 rounded to nearest in fp32, and the kernels convert every tap exactly before the fp32
arithmetic, so a uint8 render must be BITWISE equal to the fp32 render of that conversion (numpy's astype(np.float32) / 255.0) on the
same kernel: the direct kernel, or the staged kernel at a 2- and a 3-stage ring.  Shapes the staged kernels cannot take in uint8
(Wt % 16 != 0, a base that is not 16-byte aligned) run the direct kernel and are compared with the direct kernel on the conversion."""
import ctypes
import functools
import os

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from ml_gmpi_b200.camera import cam_params
from conftest import ROOT
from testlib import (CASES, assert_bitwise, assert_class_88_behind_plane_25, case, dev, early_stop_stats, footprints, forced_kernel,
                     forward_desc, headline_case, kernel_fixture, misaligned, native_vs_fp32, render_fwd, skip_stats)

pytestmark = pytest.mark.gpu
TAUS = [None, 0.0, 2.0 ** -24, 1e-3]
variant = kernel_fixture("direct", "staged2", "staged3")


def quantize(rgba):
    return np.clip(np.rint(np.asarray(rgba, np.float64) * 255.0), 0, 255).astype(np.uint8)


def converted(u8):
    return u8.astype(np.float32) / 255.0


def _mpi(u8, native, misalign=False):
    """The MPI of uint8 codes `u8` on the device: native (GMPI_MPI_U8) or its fp32 conversion."""
    rgba = torch.from_numpy(np.ascontiguousarray(u8 if native else converted(u8))).to(dev())
    return dict(rgba=misaligned(rgba, 8) if misalign else rgba)


def run_pair(c, u8, variant, misalign=False, **kw):
    """uint8 render and the fp32 render of its conversion, on the kernel the uint8 call gets under `variant`."""
    return native_vs_fp32(c, _mpi(u8, True, misalign), _mpi(u8, False, misalign), variant, **kw)


def test_device_conversion_is_exact_for_every_code():
    out = torch.empty(256, device=dev())
    _lib.check(_lib.load().gmpi_debug_u8_codes(out.data_ptr(), None))
    torch.cuda.synchronize()
    exact = np.arange(256, dtype=np.uint8).astype(np.float32) / 255.0
    assert np.array_equal(out.cpu().numpy().view(np.uint32), exact.view(np.uint32))
    host = np.zeros(256, np.float32)
    _lib.check(_lib.load().gmpi_debug_u8_codes_host(host.ctypes.data))
    assert np.array_equal(host.view(np.uint32), exact.view(np.uint32))
    x = torch.randint(0, 256, (1 << 16,), dtype=torch.uint8, device=dev())
    assert np.array_equal(g.unorm8_to_float(x).cpu().numpy().view(np.uint32), exact[x.cpu().numpy()].view(np.uint32))


@pytest.mark.parametrize("name", CASES)
def test_u8_render_is_bitwise_the_conversion_render(name, variant):
    """Every golden fixture and synthetic case (expanded; the factored cases' expanded stack), align_corners both ways, non-square,
    partial tiles, N = 1 / 2 / 512, view_group > 1, uint8 video with both roundings) with early stop off and at tau = 0, 2^-24, 1e-3:
    colour, depth and flags bitwise."""
    c = case(name)
    u8 = quantize(c["rgba"])
    for kw in [{}] + ([dict(u8_round=True)] if c.get("video") else []):
        for tau in TAUS:
            h, f, _ = run_pair(c, u8, variant, tau=tau, **kw)
            assert_bitwise(h, f, (name, variant, tau, kw))


@pytest.mark.parametrize("name", ["small", "factored", "uint8"])
def test_u8_render_with_cam_rays_and_view_groups(name, variant):
    c = case(name)
    u8 = quantize(c["rgba"])
    V, _, H, W = c["ray_dir"].shape
    cs = synth.make_case(n_planes=2, tex=8, img=H, n_mpi=V, seed=3)
    cam = cam_params(cs.c2w, 1.1 * W, H, W).to(dev())
    for tau in (None, 1e-3):
        h, f, _ = run_pair(c, u8, variant, cam=cam, tau=tau)
        assert_bitwise(h, f, (name, variant, tau, "cam"))
    one = dict(c, rgba=c["rgba"][:1], view2mpi=np.zeros_like(c["view2mpi"]))      # every view on one MPI: view_group = V
    h, f, _ = run_pair(one, quantize(one["rgba"]), variant, view_group=V)
    assert_bitwise(h, f, (name, variant, "view_group"))


def test_u8_fused_gather_frames(variant):
    """The fused-gather descriptor on one GPU (a device array with this rank's frame buffer): the frames are bitwise the conversion's."""
    for name in ("small", "partial_acfalse_nonsquare"):
        c = case(name)
        u8 = quantize(c["rgba"])
        for tau in (None, 1e-3):
            h, f, _ = run_pair(c, u8, variant, tau=tau, gather=True)
            assert not np.isnan(h[0]).any()
            assert_bitwise(h, f, (name, variant, tau, "gather"))


@pytest.mark.parametrize("name", ["small", "uint8", "view_group3"])
def test_host_entry_point_takes_u8_host_buffers(name):
    """gmpi_mpi_render_host_ex from uint8 host buffers == the same call on the fp32 conversion, and == the device entry point."""
    c = case(name)
    u8 = quantize(c["rgba"])
    lib = _lib.load()
    V, _, H, W = c["ray_dir"].shape
    outs = []
    for native in (True, False):
        rgba = np.ascontiguousarray(u8 if native else converted(u8))
        h = {k: np.ascontiguousarray(c[k]) for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
        flags = np.zeros(1, np.uint32)
        if c.get("video"):
            o = dict(video_rgb=np.empty((V, H, W, 3), np.uint8), video_depth=np.empty((V, H, W, 1), np.uint8))
            extra = dict(depth_near=0.9, depth_range=np.float32(0.3).item())
        else:
            o = dict(color=np.empty((V, 3, H, W), np.float32), depth=np.empty((V, 1, H, W), np.float32))
            extra = {}
        opts = _lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | (_lib.OPT_MPI_U8 if native else 0)
        d = _lib.make_desc(options=opts, M=u8.shape[0], V=V, N=u8.shape[1], Ht=u8.shape[-2], Wt=u8.shape[-1], H=H, W=W,
                           flags=flags.ctypes.data, **extra, **{k: v.ctypes.data for k, v in {**h, "rgba": rgba, **o}.items()})
        _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0))
        outs.append(tuple(o.values()) + (flags.view(np.int32),))
    assert_bitwise(outs[0], outs[1], name)
    assert_bitwise(outs[0], render_fwd(c, _mpi(u8, True), view_group=1), (name, "device entry point"))


def _shift_footprints(c, lo, hi):
    """{shift: count} of the (tile, plane) stages whose fp32 box is staged (mode 0) with a width need in [lo, hi], by the offset of
    the fp32 box origin from the multiple of 16 the uint8 box starts at (0, 4, 8, 12)."""
    f = footprints(c)
    sel = (f["mode"] == 0) & (f["need_w"] >= lo) & (f["need_w"] <= hi)
    return {s: int((sel & (f["bx0"] % 16 == s)).sum()) for s in (0, 4, 8, 12)}


@pytest.mark.parametrize("stages,shape", [pytest.param("staged2", "limit", id="staged2"), pytest.param("staged3", "limit", id="staged3"),
                                          pytest.param("staged2", "headline", id="staged2-headline_96x1024_equal_weight"),
                                          pytest.param("staged3", "headline", id="staged3-headline_96x1024_equal_weight")])
def test_u8_at_the_widest_box_class_at_every_shift(stages, shape):
    """Footprints at the widest class (width need 81..88, class 88) whose fp32 box starts 0, 4, 8 and 12 texels past a multiple of 16:
    the uint8 kernel stages a 112-wide box from that multiple and decides fast / generic body exactly as fp32 does.  "headline": 96 x
    1024^2 with equal-weight alpha, where those footprints lie on planes that reach the render."""
    c = case("band_89_96") if shape == "limit" else headline_case()
    counts = _shift_footprints(c, 81, 88)
    assert all(n > 0 for n in counts.values()), counts
    if shape == "headline":
        assert_class_88_behind_plane_25(c)
    u8 = quantize(c["rgba"])
    with forced_kernel(stages):
        for tau in (None, 1e-3):
            h, f, fell_back = run_pair(c, u8, stages, tau=tau)
            assert not fell_back
            assert_bitwise(h, f, (stages, tau))


def test_narrow_and_misaligned_u8_take_the_direct_kernel():
    """Wt % 16 != 0 (with Wt % 4 == 0) or a base 8 bytes off a 16-byte boundary: the plan query says why, the C call runs the direct
    kernel natively, bitwise the direct kernel on the conversion; render_views takes the fp32 conversion instead, bitwise the render
    of unorm8_to_float(rgba)."""
    with forced_kernel("staged3"):
        c = case("small")
        u8 = quantize(c["rgba"])
        desc, _ = forward_desc(c, _mpi(u8, True, misalign=True))
        assert _lib.fwd_plan(desc) == (_lib.PLAN_DIRECT, 8)
        for tau in (None, 1e-3):
            h, f, fell_back = run_pair(c, u8, "staged3", misalign=True, tau=tau)
            assert fell_back
            assert_bitwise(h, f, ("misaligned", tau))
        n = case("partial_acfalse_nonsquare")        # texture 72 x 116: 116 % 16 == 4
        un = quantize(n["rgba"])
        desc, _ = forward_desc(n, _mpi(un, True))
        assert _lib.fwd_plan(desc) == (_lib.PLAN_DIRECT, 1)
        desc32, _ = forward_desc(n, _mpi(un, False))
        assert _lib.fwd_plan(desc32) == (_lib.PLAN_STAGED, 0)
        h, f, fell_back = run_pair(n, un, "staged3")
        assert fell_back
        assert_bitwise(h, f, "Wt % 16")
    # render_views: the fallback renders the conversion on the fp32 plan (staged here), and equals render_views of the conversion
    cs = synth.make_case(n_planes=8, tex=8, img=256, n_mpi=2, views_per_mpi=2, seed=4, last_alpha_one=True).to(dev())
    x = torch.randint(0, 256, (2, 8, 4, 64, 120), dtype=torch.uint8, generator=torch.Generator().manual_seed(9)).to(dev())
    args = (cs.dhw, cs.view2mpi, cs.ray_dir, cs.eye, cs.z_dir)
    with torch.no_grad():
        a = g.render_views(x, *args, unorm8=True)
        b = g.render_views(g.unorm8_to_float(x), *args)
    assert_bitwise(a, b, "render_views fallback")


@functools.lru_cache(maxsize=None)
def _dispatch_case():
    return synth.make_case(n_planes=16, tex=256, img=256, n_mpi=2, views_per_mpi=2, seed=7, last_alpha_one=True).to(dev())


def test_render_views_and_frames_take_u8_natively_without_an_fp32_copy():
    c = _dispatch_case()
    x = torch.from_numpy(quantize(c.rgba.cpu().numpy())).to(dev())
    f32 = g.unorm8_to_float(x)
    args = (c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir)
    with torch.no_grad():
        ref = g.render_views(f32, *args)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = g.render_views(x, *args, unorm8=True)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    outputs = sum(t.numel() * t.element_size() for t in out)
    assert peak <= outputs + (1 << 20), (peak, outputs, x.numel() * 4)       # no fp32 copy of the MPI (8 MB here)
    assert_bitwise(out, ref, "render_views")
    kw = dict(dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir)
    for extra in (dict(early_stop=1e-3), dict(video={"near": 0.9, "far": 1.2}), dict(video={"near": 0.9, "far": 1.2}, u8_round=True)):
        v = g.render_frames(rgba=x, unorm8=True, **kw, **extra)
        w = g.render_frames(rgba=f32, **kw, **extra)
        assert_bitwise(v, w, ("render_frames", extra))
    # unorm8 left at False: a uint8 tensor is upcast without scaling, as before
    with torch.no_grad():
        a = g.render_views(x, *args)
        b = g.render_views(x.float(), *args)
    assert_bitwise(a, b, "unorm8=False")
    with pytest.raises(TypeError, match="uint8"):
        g.render_views(f32, *args, unorm8=True)
    with pytest.raises(TypeError, match="uint8"):
        g.render_frames(rgba=x.half(), unorm8=True, **kw)


@pytest.mark.parametrize("stages", ["staged2", "staged3"])
def test_skip_empty_on_u8_is_bitwise(stages):
    """synth.make_head_case quantized to 8 bits: the uint8 map's bytes equal the map of the conversion, the skipping frames are bitwise
    those of the conversion (with and without skipping), and the skip and early-stop hooks report the uint8 launches."""
    d = dev()
    N, R, V = 32, 256, 3
    h = synth.make_head_case(n_planes=N, tex=R, img=R, n_mpi=1, views_per_mpi=V, seed=11).to(d)
    x = torch.from_numpy(quantize(h.rgba.cpu().numpy())).to(d)
    f32 = g.unorm8_to_float(x)
    o8, o32 = g.build_occupancy(rgba=x, unorm8=True), g.build_occupancy(rgba=f32)
    torch.cuda.synchronize()
    assert o8.nbytes == o32.nbytes and torch.equal(o8.occ, o32.occ)
    kw = dict(dhw=h.dhw, view2mpi=h.view2mpi, ray_dir=h.ray_dir, eye=h.eye, z_dir=h.z_dir, view_group=V)
    with forced_kernel(stages):
        for extra in ({}, dict(video={"near": 0.9, "far": 1.2}), dict(early_stop=1e-3)):
            a = g.render_frames(rgba=x, unorm8=True, skip_empty=o8, **kw, **extra)
            skipped, total = skip_stats()
            assert 0 < skipped < total, (skipped, total)
            if "early_stop" in extra:
                es, es_total = early_stop_stats()
                assert es_total == total and 0 < es < es_total
            b = g.render_frames(rgba=f32, skip_empty=o32, **kw, **extra)
            assert (skipped, total) == skip_stats()
            c = g.render_frames(rgba=f32, **kw, **extra)
            assert_bitwise(a, b, (stages, extra, "skip"))
            assert_bitwise(a, c, (stages, extra, "no skip"))
        a, c = g.render_frames(rgba=x, unorm8=True, skip_empty=True, **kw), g.render_frames(rgba=f32, **kw)
        assert_bitwise(a, c, (stages, "skip_empty=True"))


def test_u8_planes_against_the_reference():
    """The reference's mpi_from_plane_imgs + MPI.forward on seeded RGBA8 planes (oracle/make_golden_u8.py): the native uint8 render
    is within 2e-5 of the reference render, and bitwise the render of the reference's fp32 planes."""
    gd = np.load(os.path.join(ROOT, "tests", "golden", "u8_planes.npz"))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev())
    args = (t(gd["dhw"]), t(gd["view2mpi"]), t(gd["ray_dir"]), t(gd["eye"]), t(gd["z_dir"]))
    for v in ("direct", "staged2", "staged3"):
        with forced_kernel(v), torch.no_grad():
            color, depth = g.render_views(t(gd["rgba_u8"]), *args, align_corners=bool(gd["align_corners"]), unorm8=True)
            c32, d32 = g.render_views(t(gd["rgba"]), *args, align_corners=bool(gd["align_corners"]))
        assert_bitwise((color, depth), (c32, d32), v)
        for got, ref in ((color, gd["color"]), (depth, gd["depth"])):
            err = float(np.max(np.abs(got.cpu().numpy() - ref)) / max(float(np.max(np.abs(ref))), 1e-30))
            assert err <= 2e-5, (v, err)
