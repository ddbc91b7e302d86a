"""GPU parity tests (run on an H100: pytest -m gpu).  Everything goes through the C ABI
(ctypes) of libgmpi_mpi_render.so; the oracle and the golden fixtures are only the checkers.

Bars (SURVEY.md section 8c): max|ours-ref| / max|ref| <= 1e-4 for colour, depth and d/d rgba
(fp32); the texel coordinates (ix, iy) are bit-exact."""
import functools
import json

import numpy as np
import pytest
import torch

import mpi_oracle
import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib
from conftest import MPI_CASES, load_golden, rel_err
from testlib import (C4_YAWS, EXPECT, FULL, GEOMETRY, case, dev, each_alpha, kernel_fixture, on_device, oracle_backward, oracle_forward,
                     pixels, to_np, upstream)

pytestmark = pytest.mark.gpu
TOL = 1e-4          # the north star's bar


# Each test runs once per forward kernel: the direct gather, and the TMA-staged kernel at the ring depth it picks itself and forced
# to a 2- and a 3-stage ring (the expanded forward's two depths; the factored forward's ring is always 3 deep).  The full-size cases
# run the direct gather and the staged kernel at the ring depth it picks itself.
fwd_variant = kernel_fixture("direct", "staged", "staged2", "staged3")
fwd_variant_auto = kernel_fixture("direct", "staged")


def groups(gd, device):
    v2m = gd["view2mpi"]
    M = gd["rgba"].shape[0]
    t = lambda a: torch.from_numpy(a).to(device)
    idx = [np.nonzero(v2m == m)[0] for m in range(M)]
    return [t(gd["ray_dir"][i]) for i in idx], [t(gd["eye"][i]) for i in idx], [t(gd["z_dir"][i]) for i in idx]


@pytest.mark.parametrize("name", MPI_CASES + ["c1_full_256"])
def test_forward_matches_reference_golden(name, fwd_variant):
    gd = load_golden(name)
    d = dev()
    rays, eyes, zs = groups(gd, d)
    mpi = g.MPI(align_corners=bool(gd["align_corners"]), validate="defer")
    color, depth = mpi(batch_rgba=torch.from_numpy(gd["rgba"]).to(d), batch_dhw=torch.from_numpy(gd["dhw"]).to(d),
                       batch_ray_dir=rays, batch_eye_pos=eyes, batch_z_dir=zs, separate_background=None,
                       assert_not_out_of_last_plane=True)
    ec, ed = rel_err(color.cpu().numpy(), gd["color"]), rel_err(depth.cpu().numpy(), gd["depth"])
    assert ec <= EXPECT and ed <= EXPECT, (ec, ed)
    flags = mpi.last_flags()
    if name == "out_of_plane":
        assert flags & _lib.FLAG_LAST_PLANE_OOB
    elif name not in ("nonsquare", "tiny_2mpi_3view_acfalse"):
        assert flags == 0


@pytest.mark.parametrize("name", MPI_CASES)
def test_backward_matches_reference_autograd(name, fwd_variant):
    gd = load_golden(name)
    d = dev()
    rays, eyes, zs = groups(gd, d)
    rgba = torch.from_numpy(gd["rgba"]).to(d).requires_grad_(True)
    mpi = g.MPI(align_corners=bool(gd["align_corners"]), validate="off")
    color, depth = mpi(batch_rgba=rgba, batch_dhw=torch.from_numpy(gd["dhw"]).to(d), batch_ray_dir=rays,
                       batch_eye_pos=eyes, batch_z_dir=zs, separate_background=None)
    loss = (color * torch.from_numpy(gd["g_color"]).to(d)).sum()
    if "g_depth" in gd:
        loss = loss + (depth * torch.from_numpy(gd["g_depth"]).to(d)).sum()
    loss.backward()
    ours = rgba.grad.cpu().numpy()
    if "g_rgba" in gd:
        ref = gd["g_rgba"]
    else:   # large case: the golden holds inputs+upstream grads, the oracle (pinned on the others) the gradient
        ref = oracle_backward(gd, gd["g_color"], gd.get("g_depth"), align_corners=bool(gd["align_corners"]))
    e = rel_err(ours, ref)
    assert e <= 2e-5, e


@pytest.mark.parametrize("name", ["c1_small_64", "tiny_2mpi_3view", "tiny_2mpi_3view_acfalse", "out_of_plane", "nonsquare"])
@pytest.mark.parametrize("packed", [False, True])
def test_texel_coordinates_bit_exact(name, packed):
    gd = load_golden(name)
    d = dev()
    lib = _lib.load()
    Ht, Wt = gd["rgba"].shape[-2:]
    V, _, H, W = gd["ray_dir"].shape
    N = gd["dhw"].shape[1]
    ac = bool(gd["align_corners"])
    ref = mpi_oracle.coords(gd["view2mpi"], gd["dhw"], gd["ray_dir"], gd["eye"], Ht, Wt, ac)
    t = lambda a, dt=None: torch.from_numpy(np.ascontiguousarray(a)).to(d)
    v2m, dhw, ray, eye = t(gd["view2mpi"]), t(gd["dhw"]), t(gd["ray_dir"]), t(gd["eye"])
    out = torch.empty((V, N, 2, H, W), device=d, dtype=torch.float32)
    fn = lib.gmpi_debug_plane_coords_packed if packed else lib.gmpi_debug_plane_coords
    _lib.check(fn(v2m.data_ptr(), dhw.data_ptr(), ray.data_ptr(), eye.data_ptr(), out.data_ptr(),
                  V, N, Ht, Wt, H, W, _lib.OPT_ALIGN_CORNERS if ac else 0, None))
    torch.cuda.synchronize()
    ours = out.cpu().numpy()
    assert np.array_equal(ours.view(np.uint32), ref.view(np.uint32)), float(np.max(np.abs(ours - ref)))


def test_fast_division_equals_ieee_division():
    """The kernels divide with RN(1/b) + two FMAs; it must equal div.rn.f32 on every input."""
    d = dev()
    lib = _lib.load()
    gen = torch.Generator(device="cpu").manual_seed(7)
    n = 1 << 24
    for trial in range(4):
        bits_a = torch.randint(0, 2 ** 31 - 1, (n,), generator=gen, dtype=torch.int64)
        bits_b = torch.randint(0, 2 ** 31 - 1, (n,), generator=gen, dtype=torch.int64)
        # exponents within +-44 of 1.0 so both the fast range (2^+-40) and its fallback edges are hit
        mk = lambda bits: (((bits & 0x7FFFFF) | (((bits >> 23) % 89 + 83) << 23) | ((bits >> 30) << 31)) & 0xFFFFFFFF)
        a = mk(bits_a).to(torch.int64).numpy().astype(np.uint32).view(np.float32)
        b = mk(bits_b).to(torch.int64).numpy().astype(np.uint32).view(np.float32)
        if trial == 0:
            a[:1000] = 0.0
            b[1000:2000] = np.float32(1.0) - np.float32(2 ** -24)   # all-ones mantissa
        ta, tb = torch.from_numpy(a).to(d), torch.from_numpy(b).to(d)
        fast, ieee = torch.empty_like(ta), torch.empty_like(ta)
        _lib.check(lib.gmpi_debug_division(ta.data_ptr(), tb.data_ptr(), fast.data_ptr(), ieee.data_ptr(), n, None))
        torch.cuda.synchronize()
        assert torch.equal(fast.view(torch.int32), ieee.view(torch.int32))
        assert np.array_equal(ieee.cpu().numpy().view(np.uint32), (a / b).view(np.uint32))


def test_validate_full_raises_like_reference(fwd_variant):
    gd = load_golden("tiny_2mpi_3view")
    d = dev()
    rays, eyes, zs = groups(gd, d)
    kw = dict(batch_dhw=torch.from_numpy(gd["dhw"]).to(d), batch_ray_dir=rays, batch_eye_pos=eyes, batch_z_dir=zs,
              separate_background=None)
    mpi = g.MPI(validate="full")
    bad = torch.from_numpy(gd["rgba"]).to(d).clone()
    bad[1, 2, 3, 5, 5] = 1.5
    with pytest.raises(AssertionError, match="Expected alpha to be within"):
        mpi(batch_rgba=bad, **kw)
    good = torch.from_numpy(gd["rgba"]).to(d)
    mpi(batch_rgba=good, **kw)                      # passes
    go = load_golden("out_of_plane")
    rays, eyes, zs = groups(go, d)
    with pytest.raises(g.MPIOutOfPlaneError):
        mpi(batch_rgba=torch.from_numpy(go["rgba"]).to(d), batch_dhw=torch.from_numpy(go["dhw"]).to(d), batch_ray_dir=rays,
            batch_eye_pos=eyes, batch_z_dir=zs, separate_background=None, assert_not_out_of_last_plane=True)
    far = torch.from_numpy(gd["dhw"]).to(d).clone()
    far[:, 0, 0] = -5.0                             # a plane behind the camera, mpi.py:70
    with pytest.raises(AssertionError, match="Camera must be placed closer"):
        mpi(batch_rgba=good, batch_dhw=far, batch_ray_dir=kw["batch_ray_dir"], batch_eye_pos=kw["batch_eye_pos"],
            batch_z_dir=kw["batch_z_dir"], separate_background=None)


def test_color_minus1_1_is_fused_affine(fwd_variant):
    gd = load_golden("c1_small_64")
    d = dev()
    t = lambda a: torch.from_numpy(a).to(d)
    args = (t(gd["rgba"]), t(gd["dhw"]), t(gd["view2mpi"]), t(gd["ray_dir"]), t(gd["eye"]), t(gd["z_dir"]))
    c01, d01 = g.render_views(*args)
    c11, d11 = g.render_views(*args, color_minus1_1=True)
    assert torch.equal(c11, 2 * c01 - 1) and torch.equal(d01, d11)
    assert rel_err(c11.cpu().numpy(), gd["render_img"]) <= EXPECT     # MPIRenderer.render output, mpi_renderer.py:467
    assert rel_err(d11.cpu().numpy(), gd["render_depth"]) <= EXPECT


def test_host_buffer_entry_point():
    import ctypes
    gd = load_golden("tiny_2mpi_3view")
    lib = _lib.load()
    M, N, _, Ht, Wt = gd["rgba"].shape
    V, _, H, W = gd["ray_dir"].shape
    c = lambda a, dt=np.float32: np.ascontiguousarray(a, dtype=dt)
    rgba, v2m, dhw = c(gd["rgba"]), c(gd["view2mpi"], np.int32), c(gd["dhw"])
    ray, eye, z = c(gd["ray_dir"]), c(gd["eye"]), c(gd["z_dir"])
    color, depth = np.empty((V, 3, H, W), np.float32), np.empty((V, 1, H, W), np.float32)
    flags = np.zeros(1, np.uint32)
    p = lambda a: a.ctypes.data
    _lib.check(lib.gmpi_mpi_render_fwd_host(p(rgba), p(v2m), p(dhw), p(ray), p(eye), p(z), p(color), p(depth), p(flags),
                                            M, V, N, Ht, Wt, H, W, _lib.OPT_ALIGN_CORNERS, 0))
    assert rel_err(color, gd["color"]) <= EXPECT and rel_err(depth, gd["depth"]) <= EXPECT
    # second call reuses the cached staging buffers; then they are released
    color2, depth2 = np.empty_like(color), np.empty_like(depth)
    _lib.check(lib.gmpi_mpi_render_fwd_host(p(rgba), p(v2m), p(dhw), p(ray), p(eye), p(z), p(color2), p(depth2), p(flags),
                                            M, V, N, Ht, Wt, H, W, _lib.OPT_ALIGN_CORNERS, 0))
    assert np.array_equal(color, color2) and np.array_equal(depth, depth2)
    _lib.check(lib.gmpi_mpi_release_host_cache())


# ------------------------------------------------------------------------------------------------
# full-size checks (BASELINE.json configs) through size-independent properties + oracle on one view
# ------------------------------------------------------------------------------------------------
def _ffhq_case(N, res, V, seed=1234, device=None):
    from ml_gmpi_b200 import synth
    return synth.make_case(n_planes=N, tex=res, img=res, n_mpi=V, seed=seed, device=device)


# The full-size cases (testlib.FULL) run on two MPIs: U(0, 1) alpha, and equal-weight alpha (synth.equal_weight_alpha).  Under U(0, 1)
# alpha the transmittance falls as e^-i and planes past ~25 move the render and its gradient by less than the bar, so only the
# equal-weight MPI checks the back planes, where the widest box classes occur (tests/test_every_plane_weight.py).


def _full_case(name, alpha):
    from ml_gmpi_b200 import synth
    return synth.make_case(**FULL[name], alpha=alpha, device=dev())


@functools.lru_cache(maxsize=2)
def _oracle_forward(name, alpha):
    """(colour, depth) of every view of a FULL case, once per case for all the kernels a test runs."""
    return oracle_forward(_full_case(name, alpha))[:2]


_FULL_FWD = {(32, 256, 8): "full_32x256", (96, 512, 2): "full_96x512", (96, 1024, 1): "full_96x1024", (96, 1024, 4): "ffhq1024_batch4"}


@each_alpha("N,res,V", list(_FULL_FWD))
def test_full_size_against_oracle(N, res, V, alpha, fwd_variant_auto):
    """The BASELINE.json shapes, every view; (96, 1024, 4) is the benchmark's batch of four, whose MPIs 2 and 3 start past 2^31 and
    2^32 bytes."""
    name = _FULL_FWD[N, res, V]
    assert FULL[name]["n_mpi"] == V
    case = _full_case(name, alpha)
    color, depth = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir,
                                  check_last_plane=True)
    rc, rd = _oracle_forward(name, alpha)
    for v in range(rc.shape[0]):
        assert rel_err(color[v].cpu().numpy(), rc[v]) <= EXPECT, v
        assert rel_err(depth[v].cpu().numpy(), rd[v]) <= EXPECT, v


def test_sanity_mode_all_alpha_one_shows_first_plane(fwd_variant):
    """eval/prepare_fake_data.py:51-56: alpha==1 everywhere => the render is the warped plane 0."""
    d = dev()
    from ml_gmpi_b200 import synth
    # identity pose: every ray hits plane 0 (|u|,|v| <= 0.85 there); at oblique poses border rays miss it
    case = synth.make_case(n_planes=96, tex=512, img=512, n_mpi=1, seed=1234, device=d, yaws=[0.0], pitches=[0.0])
    rgba = case.rgba.clone()
    rgba[:, :, 3] = 1.0
    color, depth = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    first, dfirst = g.render_views(rgba[:, :1].contiguous(), case.dhw[:, :1].contiguous(), case.view2mpi, case.ray_dir,
                                   case.eye, case.z_dir)
    assert rel_err(color.cpu().numpy(), first.cpu().numpy()) <= 1e-6
    assert rel_err(depth.cpu().numpy(), dfirst.cpu().numpy()) <= 1e-6


def test_zero_alpha_renders_nothing_and_linearity_in_rgb(fwd_variant):
    d = dev()
    case = _ffhq_case(32, 256, 2, device=d)
    rgba = case.rgba.clone()
    rgba[:, :, 3] = 0.0
    color, depth = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    assert float(color.abs().max()) == 0.0 and float(depth.abs().max()) == 0.0
    a, b = case.rgba.clone(), case.rgba.clone()
    b[:, :, :3] = 0.25 * a[:, :, :3]
    ca, da = g.render_views(a, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    cb, db = g.render_views(b, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    assert rel_err(cb.cpu().numpy(), 0.25 * ca.cpu().numpy()) <= 1e-6     # colour is linear in rgb
    assert torch.equal(da, db)                                              # depth ignores rgb


def test_backward_96_planes_small_image_shared_mpi_vs_oracle(fwd_variant):
    """96 planes at 128^2 with the production alpha==1 last plane, two views accumulating into one MPI's gradient (the
    full-size C3/C5/C4 shapes are further down: test_full_size_*)."""
    d = dev()
    from ml_gmpi_b200 import synth
    case = synth.make_case(n_planes=96, tex=128, img=128, n_mpi=1, views_per_mpi=2, seed=5, device=d, last_alpha_one=True)
    rgba = case.rgba.clone().requires_grad_(True)
    color, depth = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    gc, gdp = upstream(2, 128, 128, 3, device=d)
    ((color * gc).sum() + (depth * gdp).sum()).backward()
    assert rel_err(to_np(rgba.grad), oracle_backward(case, gc, gdp)) <= 2e-5


def test_staged_falls_back_per_thread_for_non_projective_rays(fwd_variant):
    """The staged kernel estimates a tile's texel footprint from its corner rays.  With rays that are NOT a pinhole
    camera's (here: shuffled within the image, 200^2 pixels: partial tiles), taps fall outside the staged box and every such thread
    must take the direct-sampling fallback: results stay exact."""
    _edge_vs_oracle("shuffled_rays")


def test_degenerate_rays_do_not_poison_neighbours(fwd_variant):
    """ray_z == 0 (ray parallel to the planes) makes scale inf/NaN for that pixel only; those pixels render 0."""
    c = case("degenerate_rays")
    color, rc = _edge_vs_oracle("degenerate_rays")
    parallel = c["ray_dir"][:, 2] == 0                         # [V,H,W]
    assert parallel.any() and np.all(color.transpose(1, 0, 2, 3)[:, parallel] == 0) and np.all(rc.transpose(1, 0, 2, 3)[:, parallel] == 0)


def test_renderer_facade_matches_reference_render():
    """ml_gmpi_b200.renderer.MPIRenderer.render vs the reference's MPIRenderer.render output (golden c1_full_256:
    BASELINE.json configs[0], 32 planes, 256^2, identity pose), through given_yaws/given_pitches."""
    from ml_gmpi_b200.renderer import MPIRenderer
    from ml_gmpi_b200.geometry import FFHQ
    gd = load_golden("c1_full_256")
    d = dev()
    r = MPIRenderer(n_mpi_planes=32, plane_min_d=FFHQ["plane_min_d"], plane_max_d=FFHQ["plane_max_d"],
                    plan_spatial_enlarge_factor=FFHQ["enlarge_factor"], plane_distances_sample_method="inverse", cam_fov=12.6,
                    sphere_center_z=1.0, sphere_r=1.0, horizontal_mean=0.0, horizontal_std=0.289, vertical_mean=0.0,
                    vertical_std=0.127, cam_pose_n_truncated_stds=2, cam_sample_method="truncated_gaussian",
                    mpi_align_corners=True, use_confined_volume=True, device=d)
    img, depth, c2w, ang = r.render(torch.from_numpy(gd["rgba"]).to(d), 256, 256, given_yaws=torch.zeros(1, 1),
                                    given_pitches=torch.zeros(1, 1))
    assert rel_err(img.cpu().numpy(), gd["render_img"]) <= EXPECT
    assert rel_err(depth.cpu().numpy(), gd["render_depth"]) <= EXPECT
    assert np.allclose(c2w.cpu().numpy(), gd["render_c2w"], atol=1e-6) and np.allclose(ang.cpu().numpy(), gd["render_angles"])
    bad = torch.from_numpy(gd["rgba"]).to(d).clone()
    bad[0, 3, 1, 7, 7] = -0.5
    with pytest.raises(AssertionError):
        r.render(bad, 256, 256, given_yaws=torch.zeros(1, 1), given_pitches=torch.zeros(1, 1))
    # random poses from the truncated Gaussian stay inside the envelope => no out-of-plane flag
    torch.manual_seed(0)
    img, depth, c2w, ang = r.render(torch.from_numpy(gd["rgba"]).to(d).expand(4, -1, -1, -1, -1).contiguous(), 256, 256)
    assert img.shape == (4, 3, 256, 256) and ang.shape == (4, 2)


@each_alpha("fwd_variant", ["direct", "staged", "staged2", "staged3"], indirect=["fwd_variant"])
def test_every_view_of_a_batch_matches_the_oracle(fwd_variant, alpha):
    """All views (not just one) of a multi-view batch, including the most oblique pose of the synthetic set, whose tiles on
    the left image border have tall (scale 1.23) and partly out-of-texture footprints."""
    case = _full_case("full_32x256", alpha)
    color, depth = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    rc, rd = _oracle_forward("full_32x256", alpha)
    assert rel_err(to_np(color), rc) <= EXPECT and rel_err(to_np(depth), rd) <= EXPECT
    # single-plane renders isolate per-plane sampling errors that transmittance would otherwise hide
    for k in (0, 13, 26, 31):
        rg = case.rgba[:1].clone()
        a = rg[:, :, 3].clone(); rg[:, :, 3] = 0; rg[:, k, 3] = a[:, k]
        c1, d1 = g.render_views(rg, case.dhw[:1], case.view2mpi[:1], case.ray_dir[:1], case.eye[:1], case.z_dir[:1])
        r1, rd1, _ = oracle_forward(dict(rgba=rg, view2mpi=np.zeros(1, np.int32), dhw=case.dhw[:1], ray_dir=case.ray_dir[:1],
                                         eye=case.eye[:1], z_dir=case.z_dir[:1]))
        assert rel_err(to_np(c1), r1) <= EXPECT, k


def test_backward_staged_multi_tile_batch_vs_oracle(fwd_variant):
    """Backward over several tiles per view, several views per MPI (gradient accumulation across views), oblique poses,
    production alpha==1 last plane and a fully opaque middle region: staged sweep (transmittance saved by the forward) and
    two-pass direct kernel against the oracle's autograd-formula gradient."""
    d = dev()
    from ml_gmpi_b200 import synth
    case = synth.make_case(n_planes=24, tex=192, img=160, n_mpi=2, views_per_mpi=2, seed=11, device=d, last_alpha_one=True)
    base = case.rgba.clone()
    base[0, 7, 3, 40:120, 30:150] = 1.0
    rgba = base.clone().requires_grad_(True)
    color, depth = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, color_minus1_1=True)
    gc, gdp = upstream(4, 160, 160, 5, device=d)
    ((color * gc).sum() + (depth * gdp).sum()).backward()
    assert rel_err(to_np(rgba.grad), oracle_backward(case, gc, gdp, rgba=base, minus1_1=True)) <= 2e-5
    # colour-only upstream gradient (depth output unused, as in train.py:740)
    rgba2 = base.clone().requires_grad_(True)
    c2, _ = g.render_views(rgba2, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    (c2 * gc).sum().backward()
    assert rel_err(to_np(rgba2.grad), oracle_backward(case, gc, rgba=base)) <= 2e-5


# ------------------------------------------------------------------------------------------------
# BASELINE.json configs at their REAL sizes (round-1 VERDICT: the staged backward had never been compared with the oracle
# at its operating point -- 1024^2 textures, 35x16 tiles per view, a saved-transmittance tensor map over V*N slabs, tap
# hand-over across tile edges).  The upstream gradients are upstream(V, H, W, 3) of the case's views.
# ------------------------------------------------------------------------------------------------
def _oracle_grad(case, with_depth, minus1_1=False):
    """The oracle's d rgba under the case's upstream gradients."""
    V, _, H, W = case.ray_dir.shape
    return oracle_backward(case, *upstream(V, H, W, 3, with_depth), minus1_1=minus1_1)


@functools.lru_cache(maxsize=1)
def _oracle_backward(name, alpha, with_depth, minus1_1=False):
    """_oracle_grad of a FULL case, once for all the kernels a test runs."""
    return _oracle_grad(_full_case(name, alpha), with_depth, minus1_1)


def _render_and_grad(case, with_depth, minus1_1=False):
    """(colour, depth, d rgba) of the kernels under the case's upstream gradients, as numpy."""
    rgba = case.rgba.clone().requires_grad_(True)
    color, depth = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, color_minus1_1=minus1_1)
    V, _, H, W = color.shape
    gc, gdp = upstream(V, H, W, 3, with_depth, rgba.device)
    loss = (color * gc).sum()
    if with_depth:
        loss = loss + (depth * gdp).sum()
    loss.backward()
    return to_np(color), to_np(depth), to_np(rgba.grad)


def _grad_check(case, with_depth, minus1_1=False):
    return rel_err(_render_and_grad(case, with_depth, minus1_1)[2], _oracle_grad(case, with_depth, minus1_1))


def _full_grad_check(name, alpha, with_depth, minus1_1=False):
    ours = _render_and_grad(_full_case(name, alpha), with_depth, minus1_1)[2]
    return rel_err(ours, _oracle_backward(name, alpha, with_depth, minus1_1))


_AUTO = ["direct", "staged"]


@each_alpha("fwd_variant_auto", _AUTO, indirect=["fwd_variant_auto"])
def test_full_size_backward_c3_one_view_96x1024_vs_oracle(fwd_variant_auto, alpha):
    """BASELINE configs[2] (FFHQ1024 forward+backward): one 96-plane 1024^2 view, production alpha==1 last plane, colour and
    depth upstream gradients.  (gmpi/core/mpi.py:411-436 autograd; train.py:733-740.)"""
    assert _full_grad_check("c3", alpha, with_depth=True) <= EXPECT


@each_alpha("fwd_variant_auto", _AUTO, indirect=["fwd_variant_auto"])
def test_full_size_backward_ffhq1024_batch4_vs_oracle(fwd_variant_auto, alpha):
    """BASELINE configs[2] at bench.py's batch: 4 MPIs x 96 planes x 1024^2 in one 6.4 GB tensor (MPI 2 starts past 2^31 bytes, MPI
    3 past 2^32), one view each, colour and depth upstream gradients.  Each MPI's gradient against the oracle's, on its own scale."""
    ours = _render_and_grad(_full_case("ffhq1024_batch4", alpha), with_depth=True)[2]
    ref = _oracle_backward("ffhq1024_batch4", alpha, True)
    errs = [rel_err(ours[m], ref[m]) for m in range(4)]
    assert max(errs) <= EXPECT, errs


@each_alpha("fwd_variant_auto", _AUTO, indirect=["fwd_variant_auto"])
def test_full_size_backward_c5_batch4_96x512_vs_oracle(fwd_variant_auto, alpha):
    """BASELINE configs[4] per-GPU shape: M = V = 4, 96 planes, 512^2, alpha==1 last plane, colour-only upstream gradient w.r.t.
    2c-1 (what train.py:740,779 backpropagates; the depth output is discarded there)."""
    assert _full_grad_check("c5", alpha, with_depth=False, minus1_1=True) <= EXPECT


@each_alpha("fwd_variant_auto", _AUTO, indirect=["fwd_variant_auto"])
def test_full_size_backward_four_views_share_one_mpi_512_vs_oracle(fwd_variant_auto, alpha):
    """Gradient accumulation over 4 views of ONE MPI at 512^2 (the expand of train.py:733-738, train_helpers.py:181-186)."""
    assert _full_grad_check("four_views", alpha, with_depth=True) <= EXPECT


def test_the_bars_fail_on_a_slightly_wrong_problem():
    """The kernels' C3 colour and gradient on equal-weight data, checked against the oracle of a slightly wrong problem: plane N/2
    or N - 2 rolled by one texel, or plane N/2 or N - 2 left out of the gradient.  Each must fail the bar by 10x or more, so the
    full-size tests above would catch a kernel that mis-sampled, or dropped the gradient of, one plane in the back half."""
    case = _full_case("c3", "equal_weight")
    N = case.rgba.shape[1]
    color, _, grad = _render_and_grad(case, with_depth=True)
    right_c, _ = _oracle_forward("c3", "equal_weight")
    right_g = _oracle_backward("c3", "equal_weight", True)
    assert rel_err(color, right_c) <= EXPECT and rel_err(grad, right_g) <= EXPECT
    ratios = {}
    for k in (N // 2, N - 2):
        rolled = to_np(case.rgba)
        rolled[:, k] = np.roll(rolled[:, k], 1, axis=-1)
        ratios[f"plane_{k}_rolled"] = rel_err(color, oracle_forward(case, rgba=rolled)[0]) / EXPECT
        omitted = right_g.copy()
        omitted[:, k] = 0.0
        ratios[f"plane_{k}_gradient_omitted"] = rel_err(grad, omitted) / EXPECT
    print("PARITY_TEETH " + json.dumps({k: float("%.3g" % v) for k, v in ratios.items()}))
    assert all(v >= 10 for v in ratios.values()), ratios


@each_alpha("fwd_variant_auto", _AUTO, indirect=["fwd_variant_auto"])
def test_full_size_forward_c4_video_every_view_vs_oracle(fwd_variant_auto, alpha):
    """BASELINE configs[3] shape: ONE 96-plane 512^2 MPI, 15 views (one rank's share of the 120) spread over the whole
    yaw = linspace(0.5, -0.5, 120) sweep, pitch 0 (render_video.py:95-107); every view against the oracle."""
    assert len(C4_YAWS) == 15
    case = _full_case("c4_video", alpha)
    color, depth = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, check_last_plane=True)
    rc, rd = _oracle_forward("c4_video", alpha)
    for v in range(15):
        assert rel_err(to_np(color[v]), rc[v]) <= EXPECT and rel_err(to_np(depth[v]), rd[v]) <= EXPECT, v


def test_non_projective_rays_outside_the_corner_box_still_render(fwd_variant):
    """ADVICE r1: the producer's "nothing under the tile" (mode 1) comes from the four corner rays only.  Rays that are not a
    pinhole camera's can have all four tile corners miss the texture while interior pixels hit it: those pixels must still
    be rendered (and get gradient), exactly as the direct kernel and the oracle do."""
    _, rc = _edge_vs_oracle("corners_off_the_planes")
    assert float(np.abs(rc).max()) > 0.1                       # the interior really renders something


def test_plan_query_names_the_direct_kernel_cliffs():
    """The direct-kernel fallbacks are visible through gmpi_mpi_render_fwd_plan instead of only in a profile."""
    import ctypes
    lib = _lib.load()
    why = ctypes.c_uint32(0)
    assert lib.gmpi_mpi_render_fwd_plan(4, 96, 1024, 1024, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_STAGED and why.value == 0
    assert lib.gmpi_mpi_render_fwd_plan(4, 96, 1022, 1022, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 1
    assert lib.gmpi_mpi_render_fwd_plan(1, 16, 64, 64, 48, 48, None, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 2
    assert lib.gmpi_mpi_render_fwd_plan(4, 600, 1024, 1024, 1024, 1024, None, ctypes.byref(why)) == _lib.PLAN_DIRECT and why.value & 4


def test_backward_twice_and_interleaved_graphs_use_fresh_gradient_buffers():
    """Every backward allocates its own gradient buffers (zeroed by the backward kernel itself): a second backward through the same
    node (retain_graph) and two graphs alive at once must not share or re-use them."""
    from ml_gmpi_b200 import synth
    d = dev()
    case = synth.make_case(n_planes=16, tex=256, img=256, n_mpi=2, views_per_mpi=2, seed=31, device=d, last_alpha_one=True)
    rgba = case.rgba.clone().requires_grad_(True)
    c1, d1 = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)
    c2, d2 = g.render_views(rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir)      # second graph, same leaf
    (c1.sum() + d1.sum()).backward(retain_graph=True)
    g1 = rgba.grad.clone()
    rgba.grad = None
    (c1.sum() + d1.sum()).backward()                                                                 # same node again
    g1b = rgba.grad.clone()
    rgba.grad = None
    (2 * c2.sum() + 2 * d2.sum()).backward()
    g2 = rgba.grad.clone()
    assert rel_err(to_np(g1b), to_np(g1)) <= 1e-6 and rel_err(to_np(g2), 2 * to_np(g1)) <= 1e-6
    assert float(g1.abs().max()) > 0


@pytest.mark.parametrize("order", ["sorted", "interleaved", "reversed"])
def test_zero_grad_poisoned_buffer_any_view_order(order):
    """GMPI_ZERO_GRAD on the staged backward.  The buffer arrives full of NaN; views of three MPIs come sorted by MPI (MPI.forward's
    layout), interleaved or reversed, and a fourth MPI has no view; the result must equal the oracle."""
    import ctypes
    lib = _lib.load()
    d = dev()
    c = case("three_mpis_" + order)
    rgba, gc, gdp = on_device(c, "rgba", "gc", "gd")
    geo = dict(zip(GEOMETRY, on_device(c, *GEOMETRY)))
    M, N, _, Ht, Wt = rgba.shape
    V, _, H, W = geo["ray_dir"].shape
    opt = _lib.OPT_ALIGN_CORNERS
    common = dict(M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, rgba=rgba, transmittance=torch.empty((V, N, H, W), device=d),
                  stream=torch.cuda.current_stream(d).cuda_stream, **geo)
    fd = _lib.make_desc(options=opt, color=torch.empty((V, 3, H, W), device=d), depth=torch.empty((V, 1, H, W), device=d),
                        flags=torch.zeros(1, dtype=torch.int32, device=d), **common)
    _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(fd)))
    ref = oracle_backward(c, c["gc"], c["gd"])

    def bwd(g_rgba, options):
        """gmpi_mpi_render_bwd_ex straight through the C ABI into a caller-owned gradient buffer."""
        _lib.check(lib.gmpi_mpi_render_bwd_ex(ctypes.byref(_lib.make_desc(options=options, g_color=gc, g_depth=gdp, g_rgba=g_rgba,
                                                                          **common))))
        torch.cuda.synchronize()
        return g_rgba

    gbuf = bwd(torch.full_like(rgba, float("nan")), opt | _lib.OPT_ZERO_GRAD)
    assert bool(torch.isfinite(gbuf).all()), "poison survived"
    assert rel_err(to_np(gbuf), ref) <= 2e-5
    # without GMPI_ZERO_GRAD the kernel accumulates into what it is given
    gacc = bwd(torch.ones_like(rgba), opt)
    assert rel_err(to_np(gacc) - 1.0, ref) <= 2e-5


def test_zero_grad_one_mpi_many_views_poisoned_allocator_block():
    """One MPI with many views through autograd: the gradient buffer is a torch.empty block that held NaN a moment ago."""
    from ml_gmpi_b200 import synth
    d = dev()
    case = synth.make_case(n_planes=16, tex=256, img=256, n_mpi=1, views_per_mpi=6, seed=5, device=d, last_alpha_one=True)
    poison = torch.full_like(case.rgba, float("nan"))
    del poison                                                  # the next same-size torch.empty gets this block back
    assert _grad_check(case, with_depth=True) <= 2e-5


# ------------------------------------------------------------------------------------------------------------------------------
# Shapes at the edges of the staged forward's ring (fwd_variant runs each at both ring depths): one plane, kMaxPlanesStaged = 512
# planes (the plane table then ends the shared-memory allocation of either depth), partial tiles with align_corners=False
# ------------------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(maxsize=1)
def _edge_oracle(name):
    """The oracle's (colour, depth, d rgba) of a catalogue case, once for all the kernels a test runs."""
    c = case(name)
    rc, rd, _ = oracle_forward(c, align_corners=c["ac"])
    return rc, rd, oracle_backward(c, c["gc"], c["gd"], align_corners=c["ac"])


def _edge_vs_oracle(name):
    """Colour and depth (at the pixels the case checks) and d rgba under the case's upstream gradients, against the oracle.
    Returns (colour, the oracle's colour) as numpy."""
    c = case(name)
    rgba, gc, gdp = on_device(c, "rgba", "gc", "gd")
    x = rgba.requires_grad_(True)
    color, depth = g.render_views(x, *on_device(c, *GEOMETRY), align_corners=c["ac"], check_last_plane=True)
    loss = (color * gc).sum()
    if gdp is not None:
        loss = loss + (depth * gdp).sum()
    loss.backward()
    rc, rd, ref = _edge_oracle(name)
    assert rel_err(pixels(c, to_np(color)), pixels(c, rc)) <= EXPECT and rel_err(pixels(c, to_np(depth)), pixels(c, rd)) <= EXPECT
    assert rel_err(to_np(x.grad), ref) <= EXPECT
    return to_np(color), rc


def test_single_plane_vs_oracle(fwd_variant):
    _edge_vs_oracle("N1")


def test_512_planes_vs_oracle(fwd_variant):
    """N = kMaxPlanesStaged, 96^2 textures at 128^2.  Alpha is scaled down so that the back planes still show through."""
    _edge_vs_oracle("N512")


def test_partial_tiles_align_corners_false_nonsquare_vs_oracle(fwd_variant):
    """100 x 136 pixels (partial tiles in both directions for the forward's 64 x 30 and the backward's 64 x 24 tiles) cut out of
    a pinhole image, 72 x 116 textures, align_corners=False."""
    _edge_vs_oracle("partial_acfalse_nonsquare")


def test_ring_depth_policy():
    """fwd_ring_stages: 2 stages when every view has its own MPI larger than L2 (the headline forward and every training batch),
    3 when the boxes come from L2 (views sharing one MPI, or an MPI that fits)."""
    lib = _lib.load()
    dev()
    assert lib.gmpi_debug_fwd_ring_stages(4, 4, 96, 1024, 1024, 1) == 2      # 4 MPIs x 1 view, 96 x 1024^2
    assert lib.gmpi_debug_fwd_ring_stages(8, 8, 32, 256, 256, 1) == 3        # the 256^2 batch: 32 x 256^2 fits L2
    assert lib.gmpi_debug_fwd_ring_stages(1, 120, 96, 512, 512, 120) == 3    # 120 views of one 96 x 512^2 MPI, grouped
    assert lib.gmpi_debug_fwd_ring_stages(1, 120, 96, 512, 512, 1) == 3      # ... or not: the views still share the MPI
    assert lib.gmpi_debug_fwd_ring_stages(4, 4, 96, 512, 512, 1) == 2
    assert lib.gmpi_debug_fwd_ring_stages(0, 4, 96, 512, 512, 1) < 0
