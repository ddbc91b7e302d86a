"""GPU tests of fp16 MPIs (GMPI_MPI_F16) on an H100: pytest -m gpu.

An fp16 value converts to fp32 exactly and the kernels convert every tap before the fp32 arithmetic, so an fp16 render must be
BITWISE equal to the fp32 render of the upcast x.half().float() on the same kernel: the direct kernel, or the staged kernel at a
2- and a 3-stage ring.  Shapes the staged kernels cannot take in fp16 (Wt % 8 != 0, a base that is not 16-byte aligned) run the
direct kernel and are compared with the direct kernel on the upcast."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from ml_gmpi_b200.camera import cam_params
from testlib import (CASES, assert_bitwise, assert_class_88_behind_plane_25, case, dev, forced_kernel, forward_desc, headline_case,
                     kernel_fixture, limit_footprints, misaligned, native_vs_fp32, render_fwd)

pytestmark = pytest.mark.gpu
TAUS = [None, 0.0, 2.0 ** -24, 1e-3]
variant = kernel_fixture("direct", "staged2", "staged3")


def _mpi(c, half, bg=True, misalign=False):
    """The case's MPI on the device: fp16 (half) or the fp32 upcast of that fp16 MPI."""
    d = dev()
    q = lambda a: (lambda h: h if half else h.float())(torch.from_numpy(np.ascontiguousarray(a)).to(d).half())
    if c.get("factored"):
        m = dict(rgb=q(c["rgb"]), alpha=q(c["alpha"]), bg_rgb=q(c["bg"]) if bg else None)
    else:
        m = dict(rgba=q(c["rgba"]))
    if misalign:
        m = {k: None if v is None else misaligned(v, 8) for k, v in m.items()}
    return m


def run_pair(c, variant, bg=True, misalign=False, **kw):
    """fp16 render and the fp32 render of the upcast, on the kernel the fp16 call gets under `variant`."""
    return native_vs_fp32(c, _mpi(c, True, bg, misalign), _mpi(c, False, bg, misalign), variant, **kw)


@pytest.mark.parametrize("name", CASES)
def test_fp16_render_is_bitwise_the_upcast_render(name, variant):
    """Every golden fixture and synthetic case (expanded, factored with and without bg_rgb, align_corners both ways, non-square,
    partial tiles, N = 1 / 2 / 512, view_group > 1, uint8 video with both roundings) with early stop off and at tau = 0, 2^-24,
    1e-3: colour, depth and flags bitwise."""
    c = case(name)
    extra = [dict(bg=False)] if c.get("factored") else [dict(u8_round=True)] if c.get("video") else []
    for kw in [{}] + extra:
        for tau in TAUS:
            h, f, _ = run_pair(c, variant, tau=tau, **kw)
            assert_bitwise(h, f, (name, variant, tau, kw))


@pytest.mark.parametrize("name", ["small", "factored", "uint8"])
def test_fp16_render_with_cam_rays(name, variant):
    c = case(name)
    V, _, H, W = c["ray_dir"].shape
    cs = synth.make_case(n_planes=2, tex=8, img=H, n_mpi=V, seed=3)
    cam = cam_params(cs.c2w, 1.1 * W, H, W).to(dev())
    for tau in (None, 1e-3):
        h, f, _ = run_pair(c, variant, cam=cam, tau=tau)
        assert_bitwise(h, f, (name, variant, tau))


def test_unaligned_and_narrow_fp16_fall_back_to_the_direct_kernel():
    """An fp16 base 8 bytes off a 16-byte boundary, or Wt % 8 != 0 (with Wt % 4 == 0): the plan query says why, the call runs
    the direct kernel, and the output is bitwise the direct kernel's on the upcast (the staged kernel would differ in the last bits)."""
    with forced_kernel("staged3"):
        c = case("small")
        desc, _ = forward_desc(c, _mpi(c, True, misalign=True))
        assert _lib.fwd_plan(desc) == (_lib.PLAN_DIRECT, 8)
        desc32, _ = forward_desc(c, _mpi(c, False))
        assert _lib.fwd_plan(desc32) == (_lib.PLAN_STAGED, 0)
        for tau in (None, 1e-3):
            h, f, fell_back = run_pair(c, "staged3", misalign=True, tau=tau)
            assert fell_back
            assert_bitwise(h, f, ("misaligned", tau))
        n = case("partial_acfalse_nonsquare")        # texture 72 x 116: 116 % 8 == 4
        desc, _ = forward_desc(n, _mpi(n, True))
        assert _lib.fwd_plan(desc) == (_lib.PLAN_DIRECT, 1)
        desc32, _ = forward_desc(n, _mpi(n, False))
        assert _lib.fwd_plan(desc32) == (_lib.PLAN_STAGED, 0)
        h, f, fell_back = run_pair(n, "staged3")
        assert fell_back
        assert_bitwise(h, f, "Wt % 8")
    with forced_kernel("direct"):
        h32 = render_fwd(n, _mpi(n, False))
    assert_bitwise(h, h32, "Wt % 8 vs the direct kernel on the upcast")


@pytest.mark.parametrize("name", ["small", "factored", "uint8"])
def test_host_entry_point_takes_fp16_host_buffers(name):
    """gmpi_mpi_render_host_ex from fp16 host buffers == the same call on the fp32 upcast, and == the device entry point."""
    c = case(name)
    lib = _lib.load()
    V, _, H, W = c["ray_dir"].shape
    outs = []
    for half in (True, False):
        conv = lambda a: np.ascontiguousarray(a.astype(np.float16) if half else a.astype(np.float16).astype(np.float32))
        mpi = dict(rgb=conv(c["rgb"]), alpha=conv(c["alpha"]), bg_rgb=conv(c["bg"])) if c.get("factored") else dict(rgba=conv(c["rgba"]))
        ref = mpi.get("alpha", mpi.get("rgba"))
        h = {k: np.ascontiguousarray(c[k]) for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
        flags = np.zeros(1, np.uint32)
        if c.get("video"):
            o = dict(video_rgb=np.empty((V, H, W, 3), np.uint8), video_depth=np.empty((V, H, W, 1), np.uint8))
            extra = dict(depth_near=0.9, depth_range=np.float32(0.3).item())
        else:
            o = dict(color=np.empty((V, 3, H, W), np.float32), depth=np.empty((V, 1, H, W), np.float32))
            extra = {}
        opts = _lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | (_lib.OPT_MPI_F16 if half else 0)
        d = _lib.make_desc(options=opts, M=ref.shape[0], V=V, N=ref.shape[1], Ht=ref.shape[-2], Wt=ref.shape[-1], H=H, W=W,
                           flags=flags.ctypes.data, **extra, **{k: v.ctypes.data for k, v in {**h, **mpi, **o}.items()})
        _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0))
        outs.append(tuple(o.values()) + (flags.view(np.int32),))
    assert_bitwise(outs[0], outs[1], name)
    assert_bitwise(outs[0], render_fwd(c, _mpi(c, True), view_group=1), (name, "device entry point"))


def test_range_flags_match_the_fp32_check_of_the_upcast():
    d = dev()
    for shape in ((2, 3, 4, 8, 16), (1, 2, 4, 5, 5)):       # vector (slab % 8 == 0, aligned) and scalar kernels
        base = torch.rand(shape, generator=torch.Generator().manual_seed(1)).half().to(d)
        cases = {"in range": base.clone()}
        x = base.clone(); x[0, 1, 2, 3, 4] = 1.0009765625; cases["next half above 1"] = x
        x = base.clone(); x[-1, -1, 3, 0, 1] = -0.5; cases["negative alpha"] = x
        x = base.clone(); x[0, 0, 3, 2, 2] = float("nan"); cases["NaN alpha"] = x
        x = base.clone(); x[0, 0, 1, 2, 2] = float("nan"); cases["NaN colour"] = x
        x = base.clone(); x[0, 0, 0, 0, 0] = -0.0; cases["-0"] = x
        for what, x in cases.items():
            assert x.dtype == torch.float16
            f16, f32 = torch.zeros(1, dtype=torch.int32, device=d), torch.zeros(1, dtype=torch.int32, device=d)
            g.check_range(x, f16)
            g.check_range(x.float(), f32)
            assert int(f16.item()) == int(f32.item()), (shape, what, int(f16.item()), int(f32.item()))
        assert int(f32.item()) == 0
        f = torch.zeros(1, dtype=torch.int32, device=d)
        g.check_range(cases["negative alpha"], f)
        assert int(f.item()) == _lib.FLAG_ALPHA_RANGE | _lib.FLAG_RGBA_RANGE


@functools.lru_cache(maxsize=None)
def _dispatch_case():
    return synth.make_case(n_planes=16, tex=256, img=256, n_mpi=2, views_per_mpi=2, seed=7, last_alpha_one=True).to(dev())


def test_render_views_passes_fp16_natively_without_an_fp32_copy():
    c = _dispatch_case()
    x16 = c.rgba.half()
    args = (c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir)
    with torch.no_grad():
        ref = g.render_views(x16.float(), *args)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = g.render_views(x16, *args)
        torch.cuda.synchronize()
        peak = torch.cuda.max_memory_allocated() - base
    outputs = sum(t.numel() * t.element_size() for t in out)
    assert peak <= outputs + (1 << 20), (peak, outputs, x16.numel() * 4)       # no fp32 copy of the MPI (8 MB here)
    assert_bitwise(out, ref, "render_views")
    f = dict(rgb=x16[:, 0, :3].contiguous(), alpha=x16[:, :, 3:4].contiguous())
    with torch.no_grad():
        a = g.render_views_factored(f["rgb"], f["alpha"], *args)
        b = g.render_views_factored(f["rgb"].float(), f["alpha"].float(), *args)
        v = g.render_frames(rgba=x16, dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir, early_stop=1e-3)
        w = g.render_frames(rgba=x16.float(), dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir, early_stop=1e-3)
    assert_bitwise(a, b, "render_views_factored")
    assert_bitwise(v, w, "render_frames")


def test_mpi_forward_on_fp16_matches_the_upcast():
    c = _dispatch_case()
    v2m = c.view2mpi.cpu().numpy()
    idx = [np.nonzero(v2m == m)[0] for m in range(2)]
    kw = lambda rgba: dict(batch_rgba=rgba, batch_dhw=c.dhw, batch_ray_dir=[c.ray_dir[i] for i in idx],
                           batch_eye_pos=[c.eye[i] for i in idx], batch_z_dir=[c.z_dir[i] for i in idx], separate_background=None)
    x16 = c.rgba.half()
    with torch.no_grad():
        a = g.MPI(validate="full")(**kw(x16))
        b = g.MPI(validate="full")(**kw(x16.float()))
    assert_bitwise(a, b, "MPI.forward")
    bad = x16.clone()
    bad[0, 3, 3, 5, 5] = -0.25
    with torch.no_grad(), pytest.raises(AssertionError, match="alpha"):
        g.MPI(validate="full")(**kw(bad))


def test_fp16_that_requires_grad_takes_the_upcast_path():
    c = _dispatch_case()
    gen = torch.Generator().manual_seed(2)
    gc = torch.randn((4, 3, 256, 256), generator=gen).to(dev())
    grads, outs = [], []
    for upcast in (False, True):
        x = c.rgba.half().requires_grad_(True)
        color, depth = g.render_views(x.float() if upcast else x, c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir)
        (color * gc).sum().backward()
        outs.append([color.detach().cpu().numpy(), depth.detach().cpu().numpy()])
        grads.append(x.grad.cpu().numpy())
    assert_bitwise(outs[0], outs[1], "output")
    assert grads[0].dtype == np.float16
    assert_bitwise(grads[0], grads[1], "gradient")


def test_fp16_refusals_on_device_buffers():
    """Refused with GMPI_ERR_UNSUPPORTED: together with a transmittance output, on the backward, on the classic entry points."""
    c = case("small")
    lib = _lib.load()
    desc, keep = forward_desc(c, _mpi(c, True))
    V, _, H, W = c["ray_dir"].shape
    trans = torch.empty((V, c["rgba"].shape[1], H, W), device=dev())
    desc.transmittance = trans.data_ptr()
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(desc)) == 3 and b"GMPI_MPI_F16" in lib.gmpi_last_error()
    gcol = torch.zeros((V, 3, H, W), device=dev())
    g_rgba = torch.empty(c["rgba"].shape, device=dev())
    desc.g_color, desc.g_rgba = gcol.data_ptr(), g_rgba.data_ptr()
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(desc)) == 3 and b"GMPI_MPI_F16" in lib.gmpi_last_error()
    M, N, _, Ht, Wt = c["rgba"].shape
    p = [keep[k].data_ptr() for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir", "color", "depth", "flags")]
    assert lib.gmpi_mpi_render_fwd(*p, M, V, N, Ht, Wt, H, W, _lib.OPT_MPI_F16, None) == 3
    torch.cuda.synchronize()


@pytest.mark.parametrize("stages", ["staged2", "staged3"])
@pytest.mark.parametrize("factored", [pytest.param(False, id="False"), pytest.param(True, id="True"),
                                      pytest.param("headline", id="headline_96x1024_equal_weight")])
def test_fp16_at_the_widest_box_classes(factored, stages):
    """Footprints at the widest class (width need 85..88: class 88 expanded, class 96 factored; the factored case also has footprints
    93..96, which take the generic body) whose fp16 box starts 4
    texels west of the fp32 one: the fp16 kernel stages a wider box and decides fast / generic body exactly as fp32 does, so the
    render stays bitwise the upcast's.  "headline": the same at 96 x 1024^2 with equal-weight alpha, where every box class occurs on
    planes that reach the render."""
    if factored == "headline":
        c = headline_case()
        assert_class_88_behind_plane_25(c)
        factored = False
    else:
        c = dict(case("band_89_96"), factored=factored)      # the factored forward renders its factors
        assert limit_footprints(c, 85, 88) > 0 and (not factored or limit_footprints(c, 93, 96) > 0)
    with forced_kernel(stages):
        for kw in ([{}, dict(bg=False)] if factored else [{}]):
            for tau in (None, 1e-3):
                h, f, fell_back = run_pair(c, stages, tau=tau, **kw)
                assert not fell_back
                assert_bitwise(h, f, (factored, stages, tau, kw))


def test_fp16_that_requires_grad_renders_under_no_grad():
    """Under no_grad an fp16 tensor that requires grad (an fp16 parameter) renders natively, equal to the upcast render."""
    c = _dispatch_case()
    args = (c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir)
    x = torch.nn.Parameter(c.rgba.half())
    rgb, alpha = torch.nn.Parameter(x.detach()[:, 0, :3].contiguous()), torch.nn.Parameter(x.detach()[:, :, 3:4].contiguous())
    with torch.no_grad():
        pairs = [(g.render_views(x, *args), g.render_views(x.float(), *args)),
                 (g.render_views_factored(rgb, alpha, *args), g.render_views_factored(rgb.float(), alpha.float(), *args)),
                 (g.render_frames(rgba=x, dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir),
                  g.render_frames(rgba=x.float(), dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir))]
    for a, b in pairs:
        assert_bitwise(a, b, "no_grad")
    v2m = c.view2mpi.cpu().numpy()
    idx = [np.nonzero(v2m == m)[0] for m in range(2)]
    kw = lambda rgba: dict(batch_rgba=rgba, batch_dhw=c.dhw, batch_ray_dir=[c.ray_dir[i] for i in idx],
                           batch_eye_pos=[c.eye[i] for i in idx], batch_z_dir=[c.z_dir[i] for i in idx], separate_background=None)
    with torch.no_grad():
        a = g.MPI(validate="full")(**kw(x))
        b = g.MPI(validate="full")(**kw(x.float()))
    assert_bitwise(a, b, "MPI.forward under no_grad")
