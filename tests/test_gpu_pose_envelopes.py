"""The render kernels at the edges of the pose envelopes GMPI trains on: FFHQ's and MetFaces' 2-sigma and AFHQCat's 3-sigma corners
of the truncated-Gaussian yaw / pitch distribution (synth.envelope_poses), each with its own plane table, camera sphere and fov
(geometry.FFHQ, METFACES, AFHQCAT).  Run on an H100: pytest -m gpu.

At these poses most (tile, plane) stages of the staged kernels take the generic body (the forward's per-pixel path, the backward's
fp32 red.global path) beside staged tiles of the same view, and the last plane's border taps sit at the pose limit
(tests/test_pose_envelopes.py counts them and shows the 2e-5 bar sees an error confined to them).  Every check here is one the
kernels already promise at the synthetic poses: texel coordinates bit-exact; colour, depth and d rgba within 2e-5 of the oracle;
the flag word the oracle's; the opt-in forms in their exact relation to the plain fp32 render.  Each full-size case is built and
run through the oracle once, for all the kernels a test runs."""
import functools
import json

import numpy as np
import pytest
import torch

import mpi_oracle
import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from ml_gmpi_b200.camera import cam_params, focal_from_fov
from ml_gmpi_b200.geometry import AFHQCAT, FFHQ, METFACES
from ml_gmpi_b200.mpi import unorm8_to_float
from conftest import load_golden, rel_err
from testlib import (ALPHAS, EXPECT, FACTORED_RGB_EXPECT, assert_bitwise, dev, factored_refs, forced_kernel, kernel_fixture,
                     max_plane_depth, oracle_backward, oracle_forward, to_np, upstream, video_reference)

pytestmark = pytest.mark.gpu
GEOMETRIES = {"ffhq": FFHQ, "afhqcat": AFHQCAT, "metfaces": METFACES}
# The direct kernels, or the staged forward at the ring depth it picks itself or forced to a 2- or 3-stage ring; and the staged
# forward at both ring depths (the opt-in forms' relations hold on the kernel that runs them).
variant = kernel_fixture("direct", "staged", "staged2", "staged3")
ring = kernel_fixture("staged2", "staged3")


def envelope_case(tag, N, res, views, *, alpha="uniform", seed=1234, last_alpha_one=False, scale=1.0, tex=None, rgba=True,
                  device=None, head=False):
    """One MPI per view at envelope_poses(geometry, scale)[views]."""
    y, p = synth.envelope_poses(GEOMETRIES[tag], scale)
    y, p = y[views], p[views]
    kw = dict(n_planes=N, tex=tex or res, img=res, n_mpi=len(y), yaws=y, pitches=p, geometry=GEOMETRIES[tag], seed=seed,
              device=device or dev())
    if head:
        return synth.make_head_case(**kw)
    return synth.make_case(**kw, rgba=rgba, alpha=alpha, last_alpha_one=last_alpha_one)


CORNERS, CORNERS_AND_EDGES = slice(0, 4), slice(0, 8)
# name: envelope_case arguments (geometry, planes, resolution, views)
FULL = {
    "ffhq_corners_96x1024": ("ffhq", 96, 1024, CORNERS),
    "metfaces_corners_96x1024": ("metfaces", 96, 1024, CORNERS),
    "afhqcat_corners_edges_96x512": ("afhqcat", 96, 512, CORNERS_AND_EDGES),
    # the backward's: one corner view at 1024^2 (C3-style), four MPIs of four corners at 512^2 (the C5-style batch)
    "ffhq_corner_96x1024": ("ffhq", 96, 1024, slice(3, 4)),
    "metfaces_corner_96x1024": ("metfaces", 96, 1024, slice(0, 1)),
    "afhqcat_corners_96x512": ("afhqcat", 96, 512, CORNERS),
}


@functools.lru_cache(maxsize=1)
def full_case(name, alpha):
    tag, N, res, views = FULL[name]
    return envelope_case(tag, N, res, views, alpha=alpha, last_alpha_one=True)


@functools.lru_cache(maxsize=1)
def full_oracle_forward(name, alpha):
    return oracle_forward(full_case(name, alpha), check_last_plane=True)


@functools.lru_cache(maxsize=1)
def full_oracle_backward(name, alpha):
    """d rgba of the oracle under upstream(V, H, W, 3), the upstream gradients of every backward here."""
    case = full_case(name, alpha)
    V, _, H, W = case.ray_dir.shape
    return oracle_backward(case, *upstream(V, H, W, 3))


def report(kind, **kw):
    print(kind + " " + json.dumps({k: (float("%.3g" % v) if isinstance(v, float) else v) for k, v in kw.items()}))


# ------------------------------------------------------------------------------------------------------------------------------
# texel coordinates
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("packed", [False, True])
@pytest.mark.parametrize("align_corners", [True, False])
@pytest.mark.parametrize("tag", list(GEOMETRIES))
def test_texel_coordinates_bit_exact_at_every_envelope_pose(tag, align_corners, packed):
    """All nine envelope poses, at 1 and 1.02 x the envelope, 96 planes, the geometry's texture size, 128^2 pixels."""
    lib = _lib.load()
    tex = 512 if tag == "afhqcat" else 1024
    fn = lib.gmpi_debug_plane_coords_packed if packed else lib.gmpi_debug_plane_coords
    for scale in (1.0, 1.02):
        c = envelope_case(tag, 96, 128, slice(0, 9), tex=8, scale=scale, rgba=False)
        V, _, H, W = c.ray_dir.shape
        N = c.dhw.shape[1]
        ref = mpi_oracle.coords(to_np(c.view2mpi), to_np(c.dhw), to_np(c.ray_dir), to_np(c.eye), tex, tex, align_corners)
        out = torch.empty((V, N, 2, H, W), device=dev())
        _lib.check(fn(c.view2mpi.data_ptr(), c.dhw.data_ptr(), c.ray_dir.data_ptr(), c.eye.data_ptr(), out.data_ptr(), V, N, tex, tex,
                      H, W, _lib.OPT_ALIGN_CORNERS if align_corners else 0, None))
        torch.cuda.synchronize()
        ours = to_np(out)
        assert np.array_equal(ours.view(np.uint32), ref.view(np.uint32)), (scale, float(np.nanmax(np.abs(ours - ref))))


# ------------------------------------------------------------------------------------------------------------------------------
# forward: every view against the oracle, and the flag word
# ------------------------------------------------------------------------------------------------------------------------------
def _forward_params():
    for alpha in ALPHAS:
        for name in ("ffhq_corners_96x1024", "metfaces_corners_96x1024", "afhqcat_corners_edges_96x512"):
            yield pytest.param(name, alpha, id=f"{name}-{alpha}")


@pytest.mark.parametrize("name,alpha", list(_forward_params()))
def test_forward_every_view_against_the_oracle(name, alpha):
    """Direct kernel and staged kernel at both ring depths, with the last-plane check: colour and depth of every view within 2e-5 of
    the oracle, and the oracle's flag word (0: the corners stay on the last plane)."""
    case = full_case(name, alpha)
    rc, rd, rflags = full_oracle_forward(name, alpha)
    assert rflags == 0
    for v in ("direct", "staged2", "staged3"):
        flags = torch.zeros(1, dtype=torch.int32, device=dev())
        with forced_kernel(v), torch.no_grad():
            color, depth = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, check_last_plane=True,
                                          flags=flags)
        ec = [rel_err(to_np(color[i]), rc[i]) for i in range(rc.shape[0])]
        ed = [rel_err(to_np(depth[i]), rd[i]) for i in range(rd.shape[0])]
        report("ENVELOPE_FWD", case=name, alpha=alpha, variant=v, color=max(ec), depth=max(ed))
        assert max(ec) <= EXPECT and max(ed) <= EXPECT, (v, ec, ed)
        assert int(flags.item()) == rflags, (v, int(flags.item()))


@pytest.mark.parametrize("tag", list(GEOMETRIES))
def test_last_plane_flag_at_the_pose_limit(tag, variant):
    """All nine envelope poses at 1 x (rays stay on the last plane) and 1.02 x the envelope (the corners' rays leave it): with the
    last-plane check, the kernels' flag word is the oracle's, and the render still matches it."""
    for scale in (1.0, 1.02):
        c = envelope_case(tag, 96, 256, slice(0, 9), tex=256, scale=scale, alpha="equal_weight")
        rc, rd, rflags = oracle_forward(c, check_last_plane=True)
        assert rflags == (0 if scale == 1.0 else mpi_oracle.FLAG_LAST_PLANE_OOB)
        flags = torch.zeros(1, dtype=torch.int32, device=dev())
        color, depth = g.render_views(c.rgba, c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, check_last_plane=True, flags=flags)
        assert int(flags.item()) == rflags, (scale, int(flags.item()), rflags)
        assert rel_err(to_np(color), rc) <= EXPECT and rel_err(to_np(depth), rd) <= EXPECT, scale


# ------------------------------------------------------------------------------------------------------------------------------
# backward: box and direct kernels, colour and depth upstream gradients; the deterministic backward
# ------------------------------------------------------------------------------------------------------------------------------
def _grad(case, **kw):
    x = case.rgba.clone().requires_grad_(True)
    color, depth = g.render_views(x, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, **kw)
    V, _, H, W = color.shape
    gc, gd = upstream(V, H, W, 3, device=x.device)
    ((color * gc).sum() + (depth * gd).sum()).backward()
    return to_np(x.grad)


def _backward_params():
    for alpha in ALPHAS:
        for name in ("afhqcat_corners_96x512", "ffhq_corner_96x1024", "metfaces_corner_96x1024"):
            yield pytest.param(name, alpha, id=f"{name}-{alpha}")


@pytest.mark.parametrize("name,alpha", list(_backward_params()))
def test_backward_against_the_oracle(name, alpha):
    """The staged forward with the box backward and the direct kernels, d rgba within 2e-5 of the oracle; on the AFHQCat batch also
    the deterministic backward, which must repeat bit for bit."""
    case = full_case(name, alpha)
    ref = full_oracle_backward(name, alpha)
    for v in ("direct", "staged"):
        with forced_kernel(v):
            e = rel_err(_grad(case), ref)
        report("ENVELOPE_BWD", case=name, alpha=alpha, variant=v, grad=e)
        assert e <= EXPECT, (v, e)
    if name.startswith("afhqcat"):
        a, b = _grad(case, deterministic=True), _grad(case, deterministic=True)
        e = rel_err(a, ref)
        report("ENVELOPE_BWD", case=name, alpha=alpha, variant="deterministic", grad=e)
        assert e <= EXPECT, e
        assert_bitwise(a, b, "deterministic")


# ------------------------------------------------------------------------------------------------------------------------------
# the opt-in forms at the corner poses, on the staged kernel at both ring depths
# ------------------------------------------------------------------------------------------------------------------------------
FORM_TAGS = ["afhqcat", "metfaces"]        # the two envelopes that put the most stages on the generic body, 4 corners, 96 x 512^2


@functools.lru_cache(maxsize=1)
def form_case(tag):
    return envelope_case(tag, 96, 512, CORNERS, alpha="equal_weight", seed=7)


@pytest.mark.parametrize("tag", FORM_TAGS)
def test_factored_equals_expanded_and_its_backward_matches_the_oracle(tag, ring):
    """On U(0, 1) alpha, the input of the factored tests at the synthetic poses (tests/test_gpu_features.py): d rgb sums the colour
    gradients of N - 1 planes, each carried by the box backward in units of 2^-22 of its tile's largest upstream gradient, so on
    equal-weight alpha, where every plane's share is ~1/N of the sum, that sum is only good to ~2e-4."""
    c = envelope_case(tag, 96, 512, CORNERS, seed=7)
    d = dev()
    gen = torch.Generator(device=d).manual_seed(11)
    M = c.rgba.shape[0]
    rgb, bg = torch.rand((M, 3, 512, 512), generator=gen, device=d), torch.rand((M, 3, 512, 512), generator=gen, device=d)
    alpha = c.rgba[:, :, 3:4].contiguous()
    with torch.no_grad():
        cf, df = g.render_views_factored(rgb, alpha, c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, bg_rgb=bg, check_last_plane=True,
                                         color_minus1_1=True)
        ce, de = g.render_views(g.expand_factored(rgb, alpha, bg), c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, check_last_plane=True,
                                color_minus1_1=True)
    assert_bitwise((cf, df), (ce, de), "factored != expanded")
    leaves = [t.clone().requires_grad_(True) for t in (rgb, alpha, bg)]
    color, depth = g.render_views_factored(leaves[0], leaves[1], c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, bg_rgb=leaves[2])
    gc, gd = upstream(M, 512, 512, 3, device=d)
    ((color * gc).sum() + (depth * gd).sum()).backward()
    refs = factored_refs(oracle_backward(c, gc, gd, rgba=g.expand_factored(rgb, alpha, bg)))
    e = {k: rel_err(to_np(t.grad), r) for k, t, r in zip(("rgb", "alpha", "bg"), leaves, refs)}
    report("ENVELOPE_FACTORED", tag=tag, ring=ring, **e)
    assert e["alpha"] <= EXPECT and e["bg"] <= EXPECT and e["rgb"] <= FACTORED_RGB_EXPECT, e


@pytest.mark.parametrize("tag", FORM_TAGS)
def test_fp16_and_uint8_are_bitwise_their_fp32_conversions(tag, ring):
    c = form_case(tag)
    args = (c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir)
    kw = dict(check_last_plane=True, color_minus1_1=True)
    with torch.no_grad():
        x16 = c.rgba.half()
        h = g.render_views(x16, *args, **kw)
        f = g.render_views(x16.float(), *args, **kw)
        assert_bitwise(h, f, "fp16")
        u8 = torch.from_numpy(np.clip(np.rint(to_np(c.rgba).astype(np.float64) * 255), 0, 255).astype(np.uint8)).to(c.rgba.device)
        conv = (u8.cpu().float() / 255).to(c.rgba.device)           # torch's CPU division: each quotient rounded once
        assert torch.equal(unorm8_to_float(u8), conv)
        q = g.render_views(u8, *args, unorm8=True, **kw)
        f = g.render_views(conv, *args, **kw)
        assert_bitwise(q, f, "uint8")


@pytest.mark.parametrize("tag", FORM_TAGS)
def test_skip_empty_is_bitwise_the_plain_render(tag, ring):
    c = envelope_case(tag, 96, 512, CORNERS, head=True)
    kw = dict(rgba=c.rgba, dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir, check_last_plane=True)
    for extra in ({}, dict(video={"near": GEOMETRIES[tag]["plane_min_d"], "far": GEOMETRIES[tag]["plane_max_d"]})):
        plain = g.render_frames(**kw, **extra)
        skipped = g.render_frames(**kw, **extra, skip_empty=True)
        assert_bitwise(plain, skipped, extra)


@pytest.mark.parametrize("tau", [1e-3, 0.05])
@pytest.mark.parametrize("tag", FORM_TAGS)
def test_early_stop_stays_within_its_bound(tag, tau, ring):
    """Colour in [-1, 1] within 2 tau, depth within tau x the pixel's largest plane depth, of early stop off (plus the parity slack);
    tau = 0 is bitwise early stop off."""
    c = envelope_case(tag, 96, 512, CORNERS, head=True)
    kw = dict(rgba=c.rgba, dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir)
    rc, rd = (to_np(t) for t in g.render_frames(**kw))
    assert_bitwise(g.render_frames(**kw), g.render_frames(**kw, early_stop=0.0), "tau = 0")
    gc, gd = (to_np(t) for t in g.render_frames(**kw, early_stop=tau))
    assert np.max(np.abs(gc - rc)) <= 2 * tau + 2 * EXPECT, float(np.max(np.abs(gc - rc)))
    zmax = max_plane_depth(dict(ray_dir=to_np(c.ray_dir), eye=to_np(c.eye), z_dir=to_np(c.z_dir), dhw=to_np(c.dhw),
                                view2mpi=to_np(c.view2mpi)))
    excess = np.abs(gd.astype(np.float64) - rd) - tau * zmax * (1 + 1e-5)
    assert np.max(excess) <= EXPECT * float(np.max(np.abs(rd))), float(np.max(excess))


@pytest.mark.parametrize("tag", ["afhqcat"])
def test_in_kernel_rays_and_video_epilogue(tag, ring):
    """AFHQCat's fov 13.39 and camera sphere of radius 2.7: the kernel's rays match PinholeCamera's (<= 2.5e-7) and the render from
    them is the render fed with those rays; the video epilogue with near / far 2.55 / 2.8 is render_video.py's conversion."""
    lib = _lib.load()
    geo = GEOMETRIES[tag]
    c = form_case(tag)
    V, _, H, W = c.ray_dir.shape
    cam = cam_params(c.c2w, focal_from_fov(geo["fov_deg"], W), H, W).to(dev())
    rays = torch.empty_like(c.ray_dir)
    _lib.check(lib.gmpi_debug_cam_rays(cam.data_ptr(), rays.data_ptr(), V, H, W, None))
    torch.cuda.synchronize()
    err = float((rays - c.ray_dir).abs().max())
    assert err <= 2.5e-7, err
    cf, df = g.render_frames(rgba=c.rgba, dhw=c.dhw, view2mpi=c.view2mpi, cam=cam, H=H, W=W, check_last_plane=True)
    cp, dp = g.render_views(c.rgba, c.dhw, c.view2mpi, rays, c.eye, c.z_dir, check_last_plane=True, color_minus1_1=True)
    assert_bitwise((cf, df), (cp, dp), "cam rays")
    near, far = geo["plane_min_d"], geo["plane_max_d"]
    u8, d8 = g.render_frames(rgba=c.rgba, dhw=c.dhw, view2mpi=c.view2mpi, ray_dir=c.ray_dir, eye=c.eye, z_dir=c.z_dir,
                             video={"near": near, "far": far})
    c11, d11 = g.render_views(c.rgba, c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, color_minus1_1=True)
    ref_img, ref_depth = video_reference(c11, d11, near, far)
    assert np.array_equal(to_np(u8), ref_img) and np.array_equal(to_np(d8), ref_depth)
    assert int(ref_depth.max()) > 100 and int(ref_depth.min()) < 100        # depth spans 2.55-2.8, not one clipped code


# ------------------------------------------------------------------------------------------------------------------------------
# the façade against the reference's MPIRenderer.render (tests/golden/envelopes.npz)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", list(GEOMETRIES))
def test_renderer_facade_matches_the_reference_at_the_corner_poses(tag):
    from ml_gmpi_b200.renderer import MPIRenderer
    z = load_golden("envelopes")
    f = lambda k: z[f"{tag}_{k}"]
    geo = GEOMETRIES[tag]
    shape = tuple(int(s) for s in f("render_rgba_shape"))
    rgba = torch.from_numpy(np.random.default_rng(int(f("render_rgba_seed"))).random(shape, dtype=np.float32)).to(dev())
    r = MPIRenderer(n_mpi_planes=shape[1], plane_min_d=geo["plane_min_d"], plane_max_d=geo["plane_max_d"],
                    plan_spatial_enlarge_factor=geo["enlarge_factor"], plane_distances_sample_method=geo["distance_method"],
                    cam_fov=geo["fov_deg"], sphere_center_z=geo["sphere_center"][2], sphere_r=geo["sphere_r"], horizontal_mean=geo["h_mean"],
                    horizontal_std=geo["h_std"], vertical_mean=geo["v_mean"], vertical_std=geo["v_std"],
                    cam_pose_n_truncated_stds=geo["n_truncated_stds"], cam_sample_method="truncated_gaussian", mpi_align_corners=True,
                    use_confined_volume=geo["confined"], device=dev())
    np.testing.assert_allclose(r.static_mpi_plane_dhws.numpy(), f("render_dhw"), rtol=2e-6)
    y, p = synth.envelope_poses(geo)
    res = f("render_img").shape[-1]
    img, depth, c2w, ang = r.render(rgba, res, res, given_yaws=torch.from_numpy(y[:4]).view(-1, 1),
                                    given_pitches=torch.from_numpy(p[:4]).view(-1, 1))
    e = dict(img=rel_err(to_np(img), f("render_img")), depth=rel_err(to_np(depth), f("render_depth")))
    report("ENVELOPE_FACADE", tag=tag, **e)
    assert e["img"] <= EXPECT and e["depth"] <= EXPECT, e
    assert np.allclose(to_np(c2w), f("render_c2w"), atol=1e-6) and np.array_equal(to_np(ang), f("render_angles"))
