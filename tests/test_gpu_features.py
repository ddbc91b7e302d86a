"""GPU tests of the rows SURVEY.md 8(f) calls "next" (N1, N2) -- every feature against the unchanged base path or the
reference's own lines, through the C ABI's descriptor entry points:

  N1  factored MPI (shared colour + per-plane alpha, networks_cond_on_pos_enc.py:950-975) forward and backward == the
      expanded stack; view-grouped tile order (views sharing one MPI) == the default order;
  N2  video epilogue (uint8 HWC colour + normalised depth) == render_video.py:118-126 applied to the fp32 outputs;
      torchvision-rounding variant == fid_evaluation.py:125-130's save_image conversion; in-kernel ray generation (cam) ==
      PinholeCamera's rays to the last ulp or two, and the render from them == the parity-mode render fed with those rays;
  host entry point with the factored / cam / video forms == the device entry point.
"""
import ctypes

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from ml_gmpi_b200.camera import PinholeCamera, cam_params, focal_from_fov
from ml_gmpi_b200.geometry import FFHQ
from conftest import rel_err
from testlib import (EXPECT, FACTORED_RGB_EXPECT, dev, kernel_fixture, oracle_backward, oracle_forward, to_np, upstream,
                     video_reference)

pytestmark = pytest.mark.gpu


# Direct gather, or the TMA-staged forward at the ring depth it picks itself or forced to a 2- or 3-stage ring (expanded MPI; the
# factored forward's ring is 3 deep).
fwd_variant = kernel_fixture("direct", "staged", "staged2", "staged3")


def factored_case(n_planes, tex, img, n_mpi, views_per_mpi, seed, with_bg):
    d = dev()
    case = synth.make_case(n_planes=n_planes, tex=tex, img=img, n_mpi=n_mpi, views_per_mpi=views_per_mpi, seed=seed, device=d, rgba=False)
    gen = torch.Generator(device=d).manual_seed(seed + 1)
    rgb = torch.rand((n_mpi, 3, tex, tex), generator=gen, device=d)
    alpha = torch.rand((n_mpi, n_planes, 1, tex, tex), generator=gen, device=d)
    alpha[:, -1] = 1.0                                            # background_alpha_full, networks_cond_on_pos_enc.py:1307-1310
    bg = torch.rand((n_mpi, 3, tex, tex), generator=gen, device=d) if with_bg else None
    return case, rgb, alpha, bg


@pytest.mark.parametrize("with_bg", [False, True])
@pytest.mark.parametrize("shape", [(12, 96, 80, 2, 2), (32, 256, 256, 2, 2)])
def test_factored_forward_equals_expanded(shape, with_bg, fwd_variant):
    N, T, I, M, K = shape
    case, rgb, alpha, bg = factored_case(N, T, I, M, K, 5, with_bg)
    cf, df = g.render_views_factored(rgb, alpha, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, bg_rgb=bg,
                                     check_last_plane=True, color_minus1_1=True)
    ce, de = g.render_views(g.expand_factored(rgb, alpha, bg), case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir,
                            check_last_plane=True, color_minus1_1=True)
    assert torch.equal(cf, ce) and torch.equal(df, de)          # same taps, same weights, same order: bit-identical
    rc, rd, _ = oracle_forward(case, rgba=g.expand_factored(rgb, alpha, bg))
    assert rel_err(to_np(cf), 2 * rc - 1) <= EXPECT and rel_err(to_np(df), rd) <= EXPECT


@pytest.mark.parametrize("with_bg", [False, True])
@pytest.mark.parametrize("shape", [(12, 96, 80, 2, 2), (24, 256, 256, 2, 2)])
def test_factored_backward_equals_expanded_autograd(shape, with_bg, fwd_variant):
    N, T, I, M, K = shape
    case, rgb, alpha, bg = factored_case(N, T, I, M, K, 6, with_bg)
    d = dev()
    gc, gd = upstream(case.ray_dir.shape[0], I, I, 3, device=d)
    rgb_f, alpha_f = rgb.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    bg_f = bg.clone().requires_grad_(True) if with_bg else None
    cf, df = g.render_views_factored(rgb_f, alpha_f, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, bg_rgb=bg_f)
    ((cf * gc).sum() + (df * gd).sum()).backward()
    # the expanded path, differentiated through expand + cat by torch: d/d rgb = sum over the planes that share it
    rgb_e, alpha_e = rgb.clone().requires_grad_(True), alpha.clone().requires_grad_(True)
    bg_e = bg.clone().requires_grad_(True) if with_bg else None
    ce, de = g.render_views(g.expand_factored(rgb_e, alpha_e, bg_e), case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    ((ce * gc).sum() + (de * gd).sum()).backward()
    assert rel_err(to_np(alpha_f.grad), to_np(alpha_e.grad)) <= EXPECT
    assert rel_err(to_np(rgb_f.grad), to_np(rgb_e.grad)) <= EXPECT
    if with_bg:
        assert rel_err(to_np(bg_f.grad), to_np(bg_e.grad)) <= EXPECT
    # and against the oracle on the expanded stack: d/d rgb is the sum over the planes that share the colour image
    ref = oracle_backward(case, gc, gd, rgba=g.expand_factored(rgb, alpha, bg))
    assert rel_err(to_np(alpha_f.grad)[:, :, 0], ref[:, :, 3]) <= EXPECT
    last = N - 1 if with_bg else N
    assert rel_err(to_np(rgb_f.grad), ref[:, :last, :3].sum(1)) <= FACTORED_RGB_EXPECT


def test_view_grouped_tile_order_changes_nothing(fwd_variant):
    d = dev()
    case = synth.make_case(n_planes=16, tex=256, img=256, n_mpi=2, views_per_mpi=4, seed=8, device=d, last_alpha_one=True)
    outs = []
    for group in (1, 4, 2):
        rgba = case.rgba.clone().requires_grad_(True)
        c, dp = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, view_group=group)
        (c.sum() + 2 * dp.sum()).backward()
        outs.append((c.detach(), dp.detach(), rgba.grad))
    for c, dp, gr in outs[1:]:
        assert torch.equal(c, outs[0][0]) and torch.equal(dp, outs[0][1])
        assert rel_err(gr.cpu().numpy(), outs[0][2].cpu().numpy()) <= 1e-6      # atomics: summation order only


def test_video_epilogue_equals_reference_conversion(fwd_variant):
    d = dev()
    case = synth.make_case(n_planes=32, tex=256, img=256, n_mpi=1, views_per_mpi=5, seed=12, device=d, last_alpha_one=True,
                           yaws=np.linspace(0.5, -0.5, 5).astype(np.float32), pitches=np.zeros(5, np.float32))
    near, far = FFHQ["plane_min_d"], FFHQ["plane_max_d"]
    c, dp = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, color_minus1_1=True)
    u8, d8 = g.render_frames(rgba=case.rgba, dhw=case.dhw, view2mpi=case.view2mpi, ray_dir=case.ray_dir, eye=case.eye, z_dir=case.z_dir,
                             video={"near": near, "far": far}, view_group=5)
    ref_img, ref_depth = video_reference(c, dp, near, far)
    assert u8.shape == (5, 256, 256, 3) and d8.shape == (5, 256, 256, 1)
    assert np.array_equal(u8.cpu().numpy(), ref_img) and np.array_equal(d8.cpu().numpy(), ref_depth)
    assert 20 < int(ref_img.std()) and int(ref_depth.max()) > 100          # the frames are not trivially constant
    # torchvision save_image(normalize=True, range=(-1, 1)): clamp, (x+1)/2, *255 + 0.5, clamp, uint8 (fid_evaluation.py:125-130)
    r8, _ = g.render_frames(rgba=case.rgba, dhw=case.dhw, view2mpi=case.view2mpi, ray_dir=case.ray_dir, eye=case.eye, z_dir=case.z_dir,
                            video={"near": near, "far": far, "depth": False}, u8_round=True)
    ref = c.clamp(-1, 1).sub(-1).div(2).mul(255).add_(0.5).clamp_(0, 255).to(torch.uint8).permute(0, 2, 3, 1)
    assert torch.equal(r8, ref.contiguous())


def test_in_kernel_rays_match_the_pinhole_camera_and_render_identically(fwd_variant):
    d = dev()
    lib = _lib.load()
    H = W = 256
    case = synth.make_case(n_planes=32, tex=256, img=H, n_mpi=2, views_per_mpi=2, seed=4, device=d, last_alpha_one=True)
    focal = focal_from_fov(FFHQ["fov_deg"], W)
    cam = cam_params(case.c2w, focal, H, W).to(d)
    rays = torch.empty_like(case.ray_dir)
    _lib.check(lib.gmpi_debug_cam_rays(cam.data_ptr(), rays.data_ptr(), 4, H, W, None))
    torch.cuda.synchronize()
    # (a) the kernel's rays vs PinholeCamera.generate_rays (fp64 camera ray -> fp32 -> fp32 matmul): the matmul's summation order is
    # the library's, so allow a couple of ulp; the camera-space stage itself is bit-exact (checked through an identity rotation)
    err = (rays - case.ray_dir).abs().max().item()
    assert err <= 2.5e-7, err
    ident = torch.eye(4, device=d).repeat(1, 1, 1)
    cam_i = cam_params(ident, focal, H, W)
    r_i = torch.empty((1, 3, H, W), device=d)
    _lib.check(lib.gmpi_debug_cam_rays(cam_i.data_ptr(), r_i.data_ptr(), 1, H, W, None))
    ref_i, _, _ = PinholeCamera(H, W, focal).generate_rays(ident)
    assert torch.equal(r_i, ref_i)
    # (b) the fast-mode render == the parity-mode render fed with the kernel's own rays (everything downstream is shared)
    cf, df = g.render_frames(rgba=case.rgba, dhw=case.dhw, view2mpi=case.view2mpi, cam=cam, H=H, W=W, check_last_plane=True)
    cp, dp = g.render_views(case.rgba, case.dhw, case.view2mpi, rays, case.eye, case.z_dir, check_last_plane=True, color_minus1_1=True)
    assert torch.equal(cf, cp) and torch.equal(df, dp)
    # (c) and it stays within the bar of the reference-ray render (different rays by an ulp: white-noise MPIs amplify it)
    cr, dr = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, color_minus1_1=True)
    assert rel_err(cf.cpu().numpy(), cr.cpu().numpy()) <= 1e-3 and rel_err(df.cpu().numpy(), dr.cpu().numpy()) <= 1e-3


def test_host_entry_point_with_factored_cam_and_video_forms():
    d = dev()
    lib = _lib.load()
    H = W = 128
    N, T = 12, 128
    case, rgb, alpha, bg = factored_case(N, T, H, 2, 2, 21, True)
    focal = focal_from_fov(FFHQ["fov_deg"], W)
    cam = cam_params(case.c2w, focal, H, W)
    near, far = FFHQ["plane_min_d"], FFHQ["plane_max_d"]
    u8, d8 = g.render_frames(rgb=rgb, alpha=alpha, bg_rgb=bg, dhw=case.dhw, view2mpi=case.view2mpi, cam=cam.to(d), H=H, W=W,
                             video={"near": near, "far": far})
    h = {k: v.cpu().contiguous() for k, v in dict(rgb=rgb, alpha=alpha, bg=bg, dhw=case.dhw, v2m=case.view2mpi, cam=cam).items()}
    o_rgb = torch.empty((4, H, W, 3), dtype=torch.uint8)
    o_dep = torch.empty((4, H, W, 1), dtype=torch.uint8)
    flags = np.zeros(1, np.uint32)
    desc = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1, M=2, V=4, N=N, Ht=T, Wt=T, H=H, W=W,
                          depth_near=float(np.float32(near)), depth_range=float(np.float32(far - near)), rgb=h["rgb"], alpha=h["alpha"],
                          bg_rgb=h["bg"], view2mpi=h["v2m"], dhw=h["dhw"], cam=h["cam"], video_rgb=o_rgb, video_depth=o_dep,
                          flags=flags.ctypes.data)
    _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(desc), 0))
    assert flags[0] == 0
    assert torch.equal(o_rgb, u8.cpu()) and torch.equal(o_dep, d8.cpu())
    _lib.check(lib.gmpi_mpi_release_host_cache())


def test_video_service_equals_the_per_view_reference_loop():
    """service.render_video_frames (one launch, uint8 epilogue, one D2H) == generate_img's loop (render_video.py:95-126): one
    MPIRenderer.render per angle, then the numpy conversion lines."""
    from ml_gmpi_b200 import service
    from ml_gmpi_b200.renderer import MPIRenderer
    d = dev()
    N, T, I = 32, 256, 256
    r = MPIRenderer(n_mpi_planes=N, plane_min_d=FFHQ["plane_min_d"], plane_max_d=FFHQ["plane_max_d"],
                    plan_spatial_enlarge_factor=FFHQ["enlarge_factor"], plane_distances_sample_method="inverse", cam_fov=12.6,
                    sphere_center_z=1.0, sphere_r=1.0, horizontal_mean=0.0, horizontal_std=0.289, vertical_mean=0.0,
                    vertical_std=0.127, cam_pose_n_truncated_stds=2, cam_sample_method="truncated_gaussian",
                    mpi_align_corners=True, use_confined_volume=True, device=d)
    gen = torch.Generator(device=d).manual_seed(3)
    mpi = torch.rand((1, N, 4, T, T), generator=gen, device=d)
    mpi[:, -1, 3] = 1.0
    angles = service.sweep_angles(6, True)
    near, far = 0.95, 1.12                                                 # curriculums.py:110-111 ray_start / ray_end
    dhw = r.static_mpi_plane_dhws.to(d).reshape(1, N, 3)
    img, depth = service.render_video_frames(mpi, dhw, angles, img_size=I, fov_deg=12.6, ray_start=near, ray_end=far,
                                             sphere_center=r.sphere_center, sphere_r=r.sphere_r)
    assert img.shape == (6, I, I, 3) and depth.shape == (6, I, I, 1)
    for i, a in enumerate(angles):
        im, dm, _, _ = r.render(mpi, I, I, horizontal_mean=a, horizontal_std=0.0, vertical_mean=0.0, vertical_std=0.0,
                                assert_not_out_of_last_plane=True)
        ref_img, ref_depth = video_reference(im, dm, near, far)
        # The service rotates the camera rays of all its views in ONE batched matmul, the loop one view at a time: cuBLAS may sum
        # the three products in a different order, the rays differ in the last ulp and a white-noise MPI turns that into a grey
        # level on a few pixels.  (With identical rays the frames are identical: test_video_epilogue_equals_reference_conversion.)
        for ours, ref in ((img[i].numpy(), ref_img[0]), (depth[i].numpy(), ref_depth[0])):
            diff = np.abs(ours.astype(np.int16) - ref.astype(np.int16))
            assert int(diff.max()) <= 1 and float((diff > 0).mean()) < 0.02, (i, int(diff.max()), float((diff > 0).mean()))
    # the fast mode (rays generated in the kernel) differs from the parity frames by at most one grey level on a few pixels
    fast, _ = service.render_video_frames(mpi, dhw, angles, img_size=I, fov_deg=12.6, ray_start=near, ray_end=far,
                                          sphere_center=r.sphere_center, sphere_r=r.sphere_r, fast_rays=True)
    diff = (fast.to(torch.int16) - img.to(torch.int16)).abs()
    assert int(diff.max()) <= 1 and float((diff > 0).float().mean()) < 0.02
