"""The cameras of the three datasets GMPI trains on (geometry.FFHQ, AFHQCAT, METFACES) at the edges of their truncated-Gaussian pose
envelopes: host geometry, oracle and torch port against the unmodified reference (tests/golden/envelopes.npz, written by
oracle/make_golden_envelopes.py), and what these poses make the staged kernels do.  CPU only.

The plane table is sized so that the envelope's corner poses just reach the last plane's edge, so at those poses the tiles' texel
footprints are the widest and tallest training produces: most (tile, plane) stages no longer fit a ring stage and take the generic
body (mode 2 of mpi_oracle.footprints: the forward's per-pixel path, the backward's fp32 red.global path), beside staged tiles in the
same view.  The census pins that the full-size GPU tests of tests/test_gpu_pose_envelopes.py reach every such path; the teeth show
that their 2e-5 bar sees an error made only inside the mode-2 stages."""
import functools

import numpy as np
import pytest
import torch

import mpi_oracle
import torch_port
from ml_gmpi_b200 import camera, geometry, synth
from conftest import load_golden, rel_err

GEOMETRIES = {"ffhq": geometry.FFHQ, "afhqcat": geometry.AFHQCAT, "metfaces": geometry.METFACES}
BAR = 2e-5                 # the GPU parity bar (tests/test_gpu_parity.py EXPECT)
TEETH = 100 * BAR
TOL = 2e-6                 # tests/test_oracle_golden.py


@functools.lru_cache(maxsize=None)
def fixture():
    return load_golden("envelopes")


def fx(tag, key):
    return fixture()[f"{tag}_{key}"]


# ------------------------------------------------------------------------------------------------------------------------------
# host geometry against the reference (tests/test_host_geometry.py's tolerances)
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", ["afhqcat", "metfaces"])
def test_plane_tables_match_reference(tag):
    for n in (8, 32, 96):
        ours = geometry.plane_dhw_table(n_planes=n, **GEOMETRIES[tag])
        ref = fx(tag, f"n{n}")
        assert ours.shape == ref.shape and ours.dtype == np.float32
        np.testing.assert_allclose(ours, ref, rtol=2e-6, atol=0)
        assert torch.equal(synth.plane_table(n, GEOMETRIES[tag]), torch.from_numpy(ours))


def test_dataset_cameras():
    """AFHQCat's camera sits 2.7 from the planes at 2.55-2.8, FFHQ's and MetFaces' at 1.0 from 0.95-1.12; the last plane of each
    table is wider than its first (the envelope's corners reach it)."""
    a, m = geometry.AFHQCAT, geometry.METFACES
    assert (a["fov_deg"], a["sphere_r"], a["sphere_center"], a["n_truncated_stds"], a["h_std"], a["v_std"]) == (13.39, 2.7, (0.0, 0.0, 2.7), 3, 0.19, 0.15)
    assert (m["fov_deg"], m["sphere_r"], m["n_truncated_stds"], m["h_std"], m["v_std"]) == (12.6, 1.0, 2, 0.339, 0.133)
    for geo in GEOMETRIES.values():
        t = synth.plane_table(96, geo).numpy()
        assert t[0, 0] == np.float32(geo["plane_min_d"]) and abs(t[-1, 0] - geo["plane_max_d"]) < 1e-6 and (t[-1, 1:] > t[0, 1:]).all()
    assert not torch.equal(synth.plane_table(32, geometry.FFHQ), synth.plane_table(32, geometry.METFACES))
    assert torch.equal(synth.plane_table(32), synth.ffhq_dhw(32))


def test_envelope_poses():
    y, p = synth.envelope_poses(geometry.AFHQCAT)
    assert y.dtype == np.float32 and y.tolist() == np.float32([-0.57, 0.57, -0.57, 0.57, -0.57, 0.57, 0, 0, 0]).tolist()
    assert p.tolist() == np.float32([-0.45, -0.45, 0.45, 0.45, 0, 0, -0.45, 0.45, 0]).tolist()
    y, p = synth.envelope_poses(geometry.FFHQ, 1.02)
    assert y[3] == np.float32(2 * 1.02 * 0.289) and p[3] == np.float32(2 * 1.02 * 0.127)
    # the default synthetic poses do not move
    c = synth.make_case(n_planes=8, tex=16, img=12, n_mpi=3, seed=1234, rgba=False)
    rng = np.random.default_rng(1234)
    assert np.array_equal(c.yaws.numpy(), rng.uniform(-0.5, 0.5, 3).astype(np.float32))
    assert torch.equal(c.dhw[0], synth.ffhq_dhw(8))


@pytest.mark.parametrize("scale", ["", "_102"])
@pytest.mark.parametrize("tag", list(GEOMETRIES))
def test_envelope_poses_and_rays_match_reference(tag, scale):
    geo = GEOMETRIES[tag]
    yaws, pitches = synth.envelope_poses(geo, 1.02 if scale else 1.0)
    assert np.array_equal(yaws, fx(tag, "yaws" + scale)) and np.array_equal(pitches, fx(tag, "pitches" + scale))
    c2w = camera.sphere_poses(torch.from_numpy(yaws), torch.from_numpy(pitches), geo["sphere_center"], geo["sphere_r"])
    np.testing.assert_allclose(c2w.numpy(), fx(tag, "c2w" + scale), atol=2e-7)
    ray, eye, z = synth.make_poses(9, 20, yaws=yaws, pitches=pitches, geometry=geo)[:3]
    np.testing.assert_allclose(ray.numpy(), fx(tag, "ray_dir" + scale), atol=2e-7)
    # from the reference's own c2w the camera's rays are the reference's bit for bit (what the render test below relies on)
    ray, eye, z = camera.PinholeCamera.from_fov(geo["fov_deg"], 20, 20).generate_rays(torch.from_numpy(fx(tag, "c2w" + scale)))
    assert np.array_equal(ray.numpy(), fx(tag, "ray_dir" + scale))
    assert np.array_equal(eye.numpy(), fx(tag, "eye" + scale)) and np.array_equal(z.numpy(), fx(tag, "z_dir" + scale))


def render_case(tag):
    """The fixture's render: the four corner views of four seeded 32-plane MPIs, one MPI per view, as oracle inputs."""
    shape = tuple(int(s) for s in fx(tag, "render_rgba_shape"))
    rgba = np.random.default_rng(int(fx(tag, "render_rgba_seed"))).random(shape, dtype=np.float32)
    res = fx(tag, "render_img").shape[-1]
    ray, eye, z = camera.PinholeCamera.from_fov(GEOMETRIES[tag]["fov_deg"], res, res).generate_rays(torch.from_numpy(fx(tag, "render_c2w")))
    dhw = np.broadcast_to(fx(tag, "render_dhw")[None], (shape[0],) + fx(tag, "render_dhw").shape).copy()
    return dict(rgba=rgba, view2mpi=np.arange(shape[0], dtype=np.int32), dhw=dhw, ray_dir=ray.numpy(), eye=eye.numpy(), z_dir=z.numpy())


@pytest.mark.parametrize("tag", list(GEOMETRIES))
def test_oracle_and_torch_port_match_reference_renders(tag):
    """MPIRenderer.render of the reference at the corner poses: colour 2c - 1 and depth.  The C oracle within test_oracle_golden's
    bar, the torch port bit for bit, and no flag: the corners stay on the last plane."""
    c = render_case(tag)
    np.testing.assert_allclose(c["dhw"][0], geometry.plane_dhw_table(n_planes=c["dhw"].shape[1], **GEOMETRIES[tag]), rtol=2e-6)
    y, p = synth.envelope_poses(GEOMETRIES[tag])
    assert np.array_equal(fx(tag, "render_angles"), np.stack([p[:4], y[:4]], -1))
    args = [c[k] for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")]
    color, depth, flags = mpi_oracle.forward(*args, check_last_plane=True, nthreads=4)
    assert rel_err(2 * color - 1, fx(tag, "render_img")) <= TOL and rel_err(depth, fx(tag, "render_depth")) <= TOL
    assert flags == 0
    t = lambda a: torch.from_numpy(a)
    views = [slice(v, v + 1) for v in range(4)]
    pc, pd = torch_port.render_views(t(c["rgba"]), t(c["dhw"]), [t(c["ray_dir"][s]) for s in views], [t(c["eye"][s]) for s in views],
                                     [t(c["z_dir"][s]) for s in views])
    assert np.array_equal((2 * pc - 1).numpy(), fx(tag, "render_img")) and np.array_equal(pd.numpy(), fx(tag, "render_depth"))


# ------------------------------------------------------------------------------------------------------------------------------
# census: the staged kernels' box modes at the shapes tests/test_gpu_pose_envelopes.py runs
# ------------------------------------------------------------------------------------------------------------------------------
CORNERS, CORNERS_AND_EDGES = slice(0, 4), slice(0, 8)
# name: (geometry, planes, resolution, views: envelope_poses indices, tiling, least share of mode-2 stages at every corner view)
CENSUS = {
    "ffhq_96x1024_fwd": ("ffhq", 96, 1024, CORNERS, mpi_oracle.FWD_TILE, 0.25),
    "ffhq_96x1024_bwd": ("ffhq", 96, 1024, slice(3, 4), mpi_oracle.BWD_TILE, 0.40),
    "metfaces_96x1024_fwd": ("metfaces", 96, 1024, CORNERS, mpi_oracle.FWD_TILE, 0.45),
    "metfaces_96x1024_bwd": ("metfaces", 96, 1024, slice(0, 1), mpi_oracle.BWD_TILE, 0.60),
    "afhqcat_96x512_fwd": ("afhqcat", 96, 512, CORNERS_AND_EDGES, mpi_oracle.FWD_TILE, 0.80),
    "afhqcat_96x512_bwd": ("afhqcat", 96, 512, CORNERS, mpi_oracle.BWD_TILE, 0.90),
}


def envelope_case(tag, N, res, views, rgba=False, alpha="uniform", seed=1234, last_alpha_one=False, scale=1.0):
    """One MPI per view at the geometry's envelope_poses[views]."""
    y, p = synth.envelope_poses(GEOMETRIES[tag], scale)
    y, p = y[views], p[views]
    return synth.make_case(n_planes=N, tex=res, img=res, n_mpi=len(y), yaws=y, pitches=p, geometry=GEOMETRIES[tag], rgba=rgba,
                           alpha=alpha, seed=seed, last_alpha_one=last_alpha_one)


@functools.lru_cache(maxsize=None)
def census_footprints(name):
    tag, N, res, views, tile, _ = CENSUS[name]
    c = envelope_case(tag, N, res, views)
    return mpi_oracle.footprints(c.view2mpi.numpy(), c.dhw.numpy(), c.ray_dir.numpy(), c.eye.numpy(), res, res, tile=tile)


@pytest.mark.parametrize("name", list(CENSUS))
def test_census_reaches_every_staged_path(name):
    tag, N, res, views, tile, least = CENSUS[name]
    f = census_footprints(name)
    mode, need_w, need_h = f["mode"], f["need_w"], f["need_h"]
    m2 = mode == 2
    wide = m2 & (need_w > 88)                                                   # the box is wider than kMaxBW
    tall = m2 & (need_w <= 88) & (-(-need_h // 4) * 4 > tile[1])                # only the rows exceed kMaxBH / kBwdMaxBH
    classes = {k: int((f["cls"] == k).sum()) for k in range(56, 96, 8)}
    share = m2.mean(axis=(1, 2, 3))                                              # per view, over all its stages
    mixed_tiles = (m2.any(-1) & (mode == 0).any(-1)).sum(axis=(1, 2))              # tiles with staged and generic planes, per view
    live = mode != 1
    print(f"CENSUS {name}: mode-2 share per view {np.round(share, 3).tolist()}, width-caused {int(wide.sum())}, "
          f"row-caused {int(tall.sum())}, classes {classes}, mixed tiles per view {mixed_tiles.tolist()}, "
          f"widest need_w {int(need_w[live].max())}, tallest need_h {int(need_h[live].max())}")
    assert wide.any() and tall.any(), (int(wide.sum()), int(tall.sum()))
    assert all(v > 0 for v in classes.values()), classes
    corners = views.start + np.arange(share.shape[0]) < 4                     # envelope_poses: the corners come first
    assert (share[corners] >= least).all(), share
    assert ((mode == 0).any(axis=(1, 2, 3)) & m2.any(axis=(1, 2, 3)))[corners].all()
    assert (mixed_tiles[corners] > 0).all(), mixed_tiles


def test_synth_pose_census_stays_mostly_staged():
    """Contrast: the synthetic U(-0.5, 0.5) x U(-0.2, 0.2) FFHQ poses of the other full-size tests put only a few percent of the
    forward's stages on the generic body."""
    c = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=1, seed=1234, rgba=False, yaws=[0.5], pitches=[0.2])
    f = mpi_oracle.footprints(c.view2mpi.numpy(), c.dhw.numpy(), c.ray_dir.numpy(), c.eye.numpy(), 1024, 1024)
    share = float((f["mode"] == 2).mean())
    print(f"CENSUS ffhq_synth_(0.5,0.2)_fwd: mode-2 share {share:.3f}")
    assert share < 0.1 < float(census_footprints("ffhq_96x1024_fwd")["mode"].__eq__(2).mean())


# ------------------------------------------------------------------------------------------------------------------------------
# the last plane's border at the envelope's edge
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tag", list(GEOMETRIES))
def test_last_plane_flag_switches_on_just_outside_the_envelope(tag):
    """At the corner poses every ray stays on the last plane (no LAST_PLANE_OOB); at 1.02 x the corner, rays leave it and the flag is
    set: the flag's edge lies at the pose limit, where the GPU tests compare the kernels' flag word with the oracle's."""
    res = 256
    for scale, expect in ((1.0, 0), (1.02, mpi_oracle.FLAG_LAST_PLANE_OOB)):
        c = envelope_case(tag, 8, res, CORNERS, rgba=True, scale=scale)
        n = lambda t: t.numpy()
        co = mpi_oracle.coords(n(c.view2mpi), n(c.dhw), n(c.ray_dir), n(c.eye), res, res)
        lo = float(co[:, -1].min())
        flags = mpi_oracle.forward(n(c.rgba), n(c.view2mpi), n(c.dhw), n(c.ray_dir), n(c.eye), n(c.z_dir), check_last_plane=True,
                                   nthreads=4)[2]
        print(f"{tag} scale {scale}: smallest last-plane texel coordinate {lo:.3f}, flags {flags}")
        assert flags == expect, (scale, flags)
        assert (lo >= 0) == (scale == 1.0)


# ------------------------------------------------------------------------------------------------------------------------------
# teeth: the 2e-5 bar sees an error confined to the mode-2 stages
# ------------------------------------------------------------------------------------------------------------------------------
TEETH_CASES = {"ffhq": (96, 1024, 3), "metfaces": (96, 1024, 0), "afhqcat": (96, 512, 0)}    # planes, resolution, corner


@functools.lru_cache(maxsize=None)
def teeth_problem(tag):
    N, res, corner = TEETH_CASES[tag]
    c = envelope_case(tag, N, res, slice(corner, corner + 1), rgba=True, alpha="equal_weight")
    geo = tuple(t.numpy() for t in (c.view2mpi, c.dhw, c.ray_dir, c.eye, c.z_dir))
    return c.rgba.numpy(), geo


def mode2_pixels(geo, k, tile):
    """[H, W] mask of the pixels whose tile takes plane k through the generic body, and the texels those pixels sample on plane k."""
    v2m, dhw, ray, eye, _ = geo
    res = ray.shape[-1]
    f = mpi_oracle.footprints(v2m, dhw, ray, eye, res, res, tile=tile)
    tiles = f["mode"][0, :, :, k] == 2
    px = np.repeat(np.repeat(tiles, tile[0], 0), 64, 1)[:res, :res]
    co = mpi_oracle.coords(v2m, dhw[:, k:k + 1], ray, eye, res, res)[0, 0]
    tex = np.zeros((res, res), bool)
    x0, y0 = np.floor(co[0][px]).astype(np.int64), np.floor(co[1][px]).astype(np.int64)
    for dy in (0, 1):
        for dx in (0, 1):
            x, y = x0 + dx, y0 + dy
            ok = (x >= 0) & (x < res) & (y >= 0) & (y < res)
            tex[y[ok], x[ok]] = True
    return px, tex


@pytest.mark.parametrize("tag", list(TEETH_CASES))
def test_bars_see_an_error_inside_the_mode2_stages(tag):
    """Equal-weight alpha, one corner view.  Plane N - 2 rolled by one texel along x only on the texels the forward's mode-2 tiles
    sample moves the oracle's colour on those tiles' pixels, and plane N - 2's gradient from only the backward's mode-2 tiles is a share
    of the whole gradient, by >= 100 x the bar.  A kernel that erred only in its generic body by that much would fail the GPU tests."""
    rgba, geo = teeth_problem(tag)
    N, res, _ = TEETH_CASES[tag]
    k = N - 2
    px, tex = mode2_pixels(geo, k, mpi_oracle.FWD_TILE)
    rolled = rgba.copy()
    rolled[0, k] = np.where(tex, np.roll(rgba[0, k], 1, axis=-1), rgba[0, k])
    right = mpi_oracle.forward(rgba, *geo, nthreads=8)[0]
    moved = mpi_oracle.forward(rolled, *geo, nthreads=8)[0]
    colour = float(np.abs(moved - right)[:, :, px].max()) / float(np.abs(right).max())       # on the mode-2 tiles' pixels only

    px_b, _ = mode2_pixels(geo, k, mpi_oracle.BWD_TILE)
    gen = np.random.default_rng(5)
    gc = gen.standard_normal((1, 3, res, res)).astype(np.float32)
    gd = gen.standard_normal((1, 1, res, res)).astype(np.float32)
    full = mpi_oracle.backward(rgba, *geo, gc, gd, nthreads=8)
    share = mpi_oracle.backward(rgba, *geo, gc * px_b, gd * px_b, nthreads=8)[:, k]
    grad = float(np.abs(share).max()) / float(np.abs(full).max())
    print(f"TEETH {tag}: plane {k}, mode-2 pixels fwd {px.mean():.3f} bwd {px_b.mean():.3f}; colour on them moved {colour / BAR:.0f} x bar, "
          f"mode-2 gradient share {grad / BAR:.0f} x bar")
    assert colour >= TEETH and grad >= TEETH, (colour / BAR, grad / BAR)
