"""GPU tests of the opt-in empty-space skipping (build_occupancy, skip_empty=...) on an H100: pytest -m gpu.

The map must equal a numpy restatement of its definition bit for bit, its fused range flags those of check_range, and every render
with skipping must be bitwise the same render without it (colour, depth, uint8 frames, flags) on the same kernel and ring depth."""
import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import synth
from conftest import MPI_CASES
from testlib import assert_bitwise, case, dev, early_stop_stats, forced_kernel, kernel_fixture, skip_stats

pytestmark = pytest.mark.gpu
B = 8
variant = kernel_fixture("direct", "staged2", "staged3")
staged = kernel_fixture("staged2", "staged3")


# ------------------------------------------------------------------------------------------------------------------------
# the map
# ------------------------------------------------------------------------------------------------------------------------
def occ_reference(alpha, colour):
    """numpy restatement: alpha [P,Ht,Wt], colour [P,3,Ht,Wt] (fp32 or fp16) -> map words [P, rows, words] (uint32)."""
    bits_a = alpha.view(np.uint32 if alpha.dtype == np.float32 else np.uint16)
    occupied = (bits_a != 0) | ~np.isfinite(colour).all(axis=1)
    P, Ht, Wt = occupied.shape
    rows, cols = -(-Ht // B), -(-Wt // B)
    pad = np.zeros((P, rows * B, cols * B), bool)
    pad[:, :Ht, :Wt] = occupied
    blocks = pad.reshape(P, rows, B, cols, B).any(axis=(2, 4))
    words = -(-cols // 32)
    full = np.zeros((P, rows, words * 32), bool)
    full[:, :, :cols] = blocks
    w = (full.reshape(P, rows, words, 32).astype(np.uint64) << np.arange(32, dtype=np.uint64)).sum(axis=-1)
    return w.astype(np.uint32)


def _specials(rgba, rng):
    """-0.0 alpha, NaN and inf colour under +0 alpha, NaN alpha, and a zero-alpha region, scattered over rgba [M,N,4,Ht,Wt]."""
    M, N, _, Ht, Wt = rgba.shape
    a = rgba[:, :, 3]
    a[rng.random(a.shape) < 0.97] = 0.0
    idx = lambda: (rng.integers(0, M), rng.integers(0, N), rng.integers(0, Ht), rng.integers(0, Wt))
    for _ in range(6):
        m, i, y, x = idx(); rgba[m, i, 3, y, x] = -0.0
        m, i, y, x = idx(); rgba[m, i, 3, y, x] = 0.0; rgba[m, i, 0, y, x] = np.nan
        m, i, y, x = idx(); rgba[m, i, 3, y, x] = 0.0; rgba[m, i, 2, y, x] = -np.inf
        m, i, y, x = idx(); rgba[m, i, 3, y, x] = np.nan
    return rgba


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("Ht,Wt", [(64, 64), (37, 83), (61, 300)])
def test_expanded_map_and_fused_flags(dtype, Ht, Wt):
    rng = np.random.default_rng(Ht * Wt)
    rgba = _specials(rng.random((2, 5, 4, Ht, Wt)).astype(np.float32), rng).astype(dtype)
    t = torch.from_numpy(rgba).to(dev())
    flags, ref_flags = (torch.zeros(1, dtype=torch.int32, device=dev()) for _ in range(2))
    occ = g.build_occupancy(rgba=t, flags=flags)
    g.check_range(t, ref_flags)
    got = occ.occ.cpu().numpy().view(np.uint32)
    ref = occ_reference(rgba[:, :, 3].reshape(-1, Ht, Wt), rgba[:, :, :3].reshape(-1, 3, Ht, Wt))
    assert np.array_equal(got[: ref.size], ref.ravel())
    assert int(flags.item()) == int(ref_flags.item()) != 0
    clean = torch.from_numpy(rng.random((1, 3, 4, Ht, Wt)).astype(dtype)).to(dev())
    f2, r2 = (torch.zeros(1, dtype=torch.int32, device=dev()) for _ in range(2))
    g.build_occupancy(rgba=clean, flags=f2)
    g.check_range(clean, r2)
    assert int(f2.item()) == int(r2.item()) == 0


@pytest.mark.parametrize("dtype", [np.float32, np.float16])
@pytest.mark.parametrize("bg", [False, True])
@pytest.mark.parametrize("Ht,Wt", [(64, 64), (37, 83)])
def test_factored_map(dtype, bg, Ht, Wt):
    rng = np.random.default_rng(7 + Ht)
    M, N = 2, 6
    rgb = rng.random((M, 3, Ht, Wt)).astype(np.float32)
    bgc = rng.random((M, 3, Ht, Wt)).astype(np.float32)
    alpha = rng.random((M, N, 1, Ht, Wt)).astype(np.float32)
    alpha[rng.random(alpha.shape) < 0.97] = 0.0
    alpha[0, 1, 0, 3, 5] = -0.0
    alpha[1, 2, 0, 7, 9] = np.nan
    rgb[0, 1, 20, 30] = np.nan
    bgc[1, 0, 11, 12] = np.inf
    rgb, bgc, alpha = rgb.astype(dtype), bgc.astype(dtype), alpha.astype(dtype)
    T = lambda x: torch.from_numpy(x).to(dev())
    occ = g.build_occupancy(rgb=T(rgb), alpha=T(alpha), bg_rgb=T(bgc) if bg else None)
    colour = np.repeat(rgb[:, None], N, axis=1)
    if bg:
        colour[:, -1] = bgc
    ref = occ_reference(alpha.reshape(-1, Ht, Wt), colour.reshape(-1, 3, Ht, Wt))
    assert np.array_equal(occ.occ.cpu().numpy().view(np.uint32)[: ref.size], ref.ravel())


# ------------------------------------------------------------------------------------------------------------------------
# renders: skipping on == skipping off, bitwise
# ------------------------------------------------------------------------------------------------------------------------
def _frames(c, skip, **kw):
    d = dev()
    T = lambda x: None if x is None else (x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(x))).to(d)
    flags = torch.zeros(1, dtype=torch.int32, device=d)
    mpi = dict(rgb=T(c["factored"][0]), alpha=T(c["factored"][1]), bg_rgb=T(c["factored"][2])) if c.get("factored") else dict(rgba=T(c["rgba"]))
    rays = dict(cam=T(c["cam"]), H=c["H"], W=c["W"]) if c.get("cam") is not None else \
        dict(ray_dir=T(c["ray_dir"]), eye=T(c["eye"]), z_dir=T(c["z_dir"]))
    with torch.no_grad():
        out = g.render_frames(dhw=T(c["dhw"]), view2mpi=T(c["view2mpi"]).int(), align_corners=c.get("ac", True), check_last_plane=True,
                              video=c.get("video"), flags=flags, view_group=c.get("view_group", 1), skip_empty=skip, **rays, **mpi, **kw)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out if o is not None] + [int(flags.item())]


def _head(n_planes=32, tex=256, img=256, n_mpi=2, views=1, seed=0, **extra):
    case = synth.make_head_case(n_planes=n_planes, tex=tex, img=img, n_mpi=n_mpi, views_per_mpi=views, seed=seed)
    c = dict(rgba=case.rgba.numpy(), view2mpi=case.view2mpi.numpy(), dhw=case.dhw.numpy(), ray_dir=case.ray_dir.numpy(),
             eye=case.eye.numpy(), z_dir=case.z_dir.numpy())
    c.update(extra)
    return c


def _factored(c, bg=True):
    rgba = torch.from_numpy(c["rgba"])
    gen = torch.Generator().manual_seed(5)
    rgb = torch.rand((rgba.shape[0], 3) + rgba.shape[-2:], generator=gen)
    c = dict(c)
    c["factored"] = (rgb, rgba[:, :, 3:4].contiguous(), torch.rand(rgb.shape, generator=gen) if bg else None)
    return c


def _transparent_but_last(seed=3):
    c = _head(n_planes=24, seed=seed)
    c["rgba"] = c["rgba"].copy()
    c["rgba"][:, :-1, 3] = 0.0
    return c


def _nan_under_zero_alpha():
    c = _head(n_planes=24, seed=4)
    c["rgba"] = c["rgba"].copy()
    c["rgba"][0, 2, 0, 100:110, 100:140] = np.nan       # under alpha 0 in front of the head: still NaN in the output
    c["rgba"][0, 2, 3, 100:110, 100:140] = 0.0
    return c


def _shuffled():
    c = _head(n_planes=24, seed=6)
    rng = np.random.default_rng(0)
    r = c["ray_dir"].copy()
    V, _, H, W = r.shape
    flat = r.reshape(V, 3, H * W)
    perm = rng.permutation(H * W)
    flat[:, :, : H * W // 2] = flat[:, :, perm[: H * W // 2]]        # half the pixels take another pixel's ray: generic bodies
    r[:, :, 40:50] = np.array([0.3, -0.2, 0.0], np.float32)[None, :, None, None]   # ray_z == 0: non-projective rows
    c["ray_dir"] = r
    return c


def _cam(video=False):
    case = synth.make_head_case(n_planes=24, tex=256, img=256, n_mpi=1, views_per_mpi=4, seed=8)
    from ml_gmpi_b200.camera import cam_params, focal_from_fov
    c = dict(rgba=case.rgba.numpy(), view2mpi=case.view2mpi.numpy(), dhw=case.dhw.numpy(), view_group=4, H=256, W=256,
             cam=cam_params(case.c2w, focal_from_fov(12.6, 256), 256, 256))
    if video:
        c["video"] = {"near": 0.88, "far": 1.12}
    return c


CASES = {
    "head": lambda: _head(),
    "head_views4_group4": lambda: _head(n_mpi=1, views=4, view_group=4),
    "head_partial_tiles": lambda: _head(img=200, seed=1),
    "head_video": lambda: _head(video={"near": 0.88, "far": 1.12}, seed=2),
    "factored_bg": lambda: _factored(_head(seed=9)),
    "factored": lambda: _factored(_head(seed=10), bg=False),
    "fp16": lambda: dict(_head(seed=11), rgba=_head(seed=11)["rgba"].astype(np.float16)),
    "fp16_factored": lambda: (lambda c: dict(c, factored=tuple(None if t is None else t.half() for t in c["factored"])))(_factored(_head(seed=12))),
    "transparent_but_last": _transparent_but_last,
    "nan_under_zero_alpha": _nan_under_zero_alpha,
    "shuffled_and_degenerate_rays": _shuffled,
    "cam_group4": lambda: _cam(),
    "cam_video": lambda: _cam(video=True),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_skip_is_bitwise_invisible(staged, name):
    c = CASES[name]()
    assert_bitwise(_frames(c, True), _frames(c, False), name)


@pytest.mark.parametrize("name", ["head", "factored_bg", "fp16", "cam_video", "shuffled_and_degenerate_rays"])
@pytest.mark.parametrize("tau", [0.0, 0.05])
def test_skip_with_early_stop_equals_early_stop_alone(staged, name, tau):
    c = CASES[name]()
    assert_bitwise(_frames(c, True, early_stop=tau), _frames(c, False, early_stop=tau), (name, tau))


@pytest.mark.parametrize("name", MPI_CASES)
def test_golden_fixtures(variant, name):
    c = case(name)
    assert_bitwise(_frames(c, True), _frames(c, False), name)


def test_nan_colour_under_zero_alpha_stays_nan(staged):
    out = _frames(_nan_under_zero_alpha(), True)
    assert np.isnan(out[0]).any()


def test_stats_random_mpi_skips_nothing_and_head_skips_the_front(staged):
    case = synth.make_case(n_planes=32, tex=256, img=256, n_mpi=2, seed=1, last_alpha_one=True)
    c = dict(rgba=case.rgba.numpy(), view2mpi=case.view2mpi.numpy(), dhw=case.dhw.numpy(), ray_dir=case.ray_dir.numpy(),
             eye=case.eye.numpy(), z_dir=case.z_dir.numpy())
    _frames(c, True)
    skipped, total = skip_stats()
    assert skipped == 0 and total > 0
    c = _head(n_planes=32)
    _frames(c, True)
    skipped, total = skip_stats()
    # planes 0..14 of 32 have alpha 0 everywhere (synth.head_alpha): most of their stages take the fast body and are empty
    assert skipped >= total * 12 // 32, (skipped, total)


@pytest.mark.parametrize("name", ["head", "fp16"])
def test_stats_of_skip_with_early_stop(staged, name):
    """A skipping launch with early stop reports the early-stop stages of the kernel that ran: it walked the stages the skip stats
    count, and armed some but not all of them without copies."""
    _frames(CASES[name](), True, early_stop=0.05)
    skipped, total = skip_stats()
    assert 0 < skipped < total, (skipped, total)
    es, es_total = early_stop_stats()
    assert es_total == total and 0 < es < es_total, (es, es_total, total)


def test_direct_kernel_skips_nothing():
    with forced_kernel("direct"):
        c = _head()
        assert_bitwise(_frames(c, True), _frames(c, False), "direct")
        assert skip_stats() == (0, 0)


def test_render_views_reuses_a_map_and_refuses_a_stale_one():
    c = _head(n_mpi=1, views=2, img=512)       # 288 tiles: the staged kernel
    d = dev()
    rgba = torch.from_numpy(c["rgba"]).to(d)
    args = [torch.from_numpy(c[k]).to(d) for k in ("dhw", "view2mpi", "ray_dir", "eye", "z_dir")]
    args[1] = args[1].int()
    occ = g.build_occupancy(rgba=rgba)
    with torch.no_grad():
        a = g.render_views(rgba, *args, skip_empty=occ)
        b = g.render_views(rgba, *args)
        assert all(torch.equal(x, y) for x, y in zip(a, b))
        rgba[0, 0, 3, 0, 0] = 1.0               # in place: the map no longer describes it
        with pytest.raises(RuntimeError, match="build it again"):
            g.render_views(rgba, *args, skip_empty=occ)
        with pytest.raises(RuntimeError, match="build it again"):
            g.render_views(rgba.clone(), *args, skip_empty=g.build_occupancy(rgba=rgba))
    with pytest.raises(RuntimeError, match="forward-only"):
        g.render_views(rgba.clone().requires_grad_(True), *args, skip_empty=True)


def _mpi_call(m, c):
    d = dev()
    rgba = torch.from_numpy(c["rgba"]).to(d)
    T = lambda k: torch.from_numpy(c[k]).to(d)
    with torch.no_grad():
        return m(batch_rgba=rgba, batch_dhw=T("dhw"), batch_ray_dir=[T("ray_dir")[i:i + 1] for i in range(rgba.shape[0])],
                 batch_eye_pos=[T("eye")[i:i + 1] for i in range(rgba.shape[0])],
                 batch_z_dir=[T("z_dir")[i:i + 1] for i in range(rgba.shape[0])], separate_background=None,
                 assert_not_out_of_last_plane=True)


@pytest.mark.parametrize("validate", ["full", "defer"])
def test_mpi_module_frames_and_exceptions(validate):
    c = _head(img=512)
    out = [_mpi_call(g.MPI(validate=validate, skip_empty=s), c) for s in (True, False)]
    assert all(torch.equal(x, y) for x, y in zip(*out))
    bad = dict(c, rgba=c["rgba"].copy())
    bad["rgba"][0, 3, 3, 10, 10] = 1.5      # alpha out of range: the same assertion with and without skipping
    msgs = []
    for s in (True, False):
        m = g.MPI(validate=validate, skip_empty=s)
        try:
            _mpi_call(m, bad)
            msgs.append(("ok", m.last_flags()))
        except AssertionError as e:
            msgs.append((type(e).__name__, str(e)))
    assert msgs[0] == msgs[1], msgs
