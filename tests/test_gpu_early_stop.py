"""GPU tests of the opt-in early ray termination (GMPI_EARLY_STOP, render_frames(early_stop=tau)) on an H100: pytest -m gpu.

Every case runs on the direct kernel and on the TMA-staged kernel forced to a 2- and a 3-stage ring.  tau = 0 must be bit-identical
to early stop off; tau > 0 must stay within the documented bound (each colour channel in [-1,1] moves by at most 2 tau, depth by at
most tau x the pixel's largest plane depth, a uint8 code by at most one) of early stop off and of the oracle, plus the parity
slack of tests/test_gpu_parity.py."""
import ctypes
import functools

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from testlib import (CASES, EXPECT, GEOMETRY, assert_bitwise, case, dev, early_stop_stats, forced_kernel, kernel_fixture,
                     max_plane_depth, on_device, oracle_forward)

pytestmark = pytest.mark.gpu
TAUS = [2.0 ** -24, 1e-3, 0.05]
variant = kernel_fixture("direct", "staged2", "staged3")


@functools.lru_cache(maxsize=None)
def oracle(name):
    c = case(name)
    color, depth, _ = oracle_forward(c, align_corners=c["ac"])
    return 2 * color - 1, depth


def render(name, early_stop=None):
    """render_frames on the case: (colour in [-1,1], depth) as numpy, or (uint8 colour, uint8 depth) for the video cases."""
    c = case(name)
    mpi = dict(zip(("rgb", "alpha", "bg_rgb"), on_device(c, "rgb", "alpha", "bg"))) if c.get("factored") else dict(rgba=on_device(c, "rgba")[0])
    video = {"near": 0.9, "far": 1.2} if c.get("video") else None
    with torch.no_grad():
        a, b = g.render_frames(**dict(zip(GEOMETRY, on_device(c, *GEOMETRY))), align_corners=c["ac"], view_group=c.get("view_group", 1),
                               video=video, early_stop=early_stop, **mpi)
    torch.cuda.synchronize()
    return a.cpu().numpy(), b.cpu().numpy()


@pytest.mark.parametrize("name", CASES)
def test_tau_zero_is_bitwise_early_stop_off(name, variant):
    off, zero = render(name), render(name, early_stop=0.0)
    assert_bitwise(off, zero, name)


def _check_bound(name, got, ref, tau, factor=1.0):
    """got vs ref within factor x the early-stop bound + the parity slack (colour in [-1,1])."""
    c = case(name)
    if c.get("video"):     # truncating uint8 codes: colour (x + 1) / 2 * 255, depth (d - 0.9) / 0.3 * 255 (render's video range)
        tol = (int(factor * tau * 255) + 1, int(factor * tau * float(np.max(max_plane_depth(c))) / 0.3 * 255) + 1)
        for x, y, k in zip(got, ref, tol):
            assert np.max(np.abs(x.astype(np.int32) - y.astype(np.int32))) <= k, (name, tau)
        return
    (gc, gd), (rc, rd) = got, ref
    assert np.max(np.abs(gc - rc)) <= factor * 2 * tau + 2 * EXPECT, (name, tau, float(np.max(np.abs(gc - rc))))
    zmax = max_plane_depth(c)
    excess = np.abs(gd.astype(np.float64) - rd) - factor * tau * zmax * (1 + 1e-5)
    assert np.max(excess) <= EXPECT * float(np.max(np.abs(rd))), (name, tau, float(np.max(excess)))


@pytest.mark.parametrize("tau", TAUS)
@pytest.mark.parametrize("name", CASES)
def test_early_stop_stays_within_its_bound(name, tau, variant):
    got = render(name, early_stop=tau)
    _check_bound(name, got, render(name), tau)
    if not case(name).get("video"):
        _check_bound(name, got, oracle(name), tau)


@pytest.mark.parametrize("tau", TAUS)
@pytest.mark.parametrize("name", ["small", "factored", "N512", "partial_acfalse_nonsquare", "c1_full_256", "alpha_one_planes"])
def test_staged_and_direct_agree_within_twice_the_bound(name, tau):
    with forced_kernel("direct"):
        direct = render(name, early_stop=tau)
    with forced_kernel("staged"):           # staged kernel at the ring depth it picks itself
        staged = render(name, early_stop=tau)
    _check_bound(name, staged, direct, tau, factor=2.0)


def _stop_planes(c, tau):
    """Per pixel [V,H,W]: the plane after which |T| <= tau (N: never), from the oracle's sampled alpha (torch_port.warp_planes)."""
    import torch_port
    N = c["rgba"].shape[1]
    v2m = c["view2mpi"]
    V, _, H, W = c["ray_dir"].shape
    rgba = torch.from_numpy(c["rgba"])[v2m].reshape(V * N, 4, *c["rgba"].shape[-2:])
    dhw = torch.from_numpy(c["dhw"])[v2m].reshape(V * N, 3)
    rep = lambda a: torch.from_numpy(a).unsqueeze(1).expand(-1, N, *a.shape[1:]).reshape(V * N, *a.shape[1:])
    _, _, alpha = torch_port.warp_planes(rgba, dhw, rep(c["eye"]), rep(c["ray_dir"]), rep(c["z_dir"]), c["ac"])
    T = torch.cumprod(1 - alpha.reshape(V, N, H, W).double(), dim=1)
    stopped = T <= tau
    return torch.where(stopped.any(1), stopped.double().argmax(1), torch.full((V, H, W), N, dtype=torch.float64)).long().numpy()


@pytest.mark.parametrize("factored", [False, True])
@pytest.mark.parametrize("stages", ["staged2", "staged3"])
def test_structured_workload_skips_stages_within_the_bound(stages, factored):
    """synth.make_head_case (opaque ellipsoidal head over ~60 % of the frame, alpha == 1 last plane): the skip counter reports
    skipped stages, the outputs meet the bound, and the workload has tiles whose warps stop at different planes and tiles where
    only some warps stop before the last plane."""
    d = dev()
    N, R, V = 32, 256, 3
    h = synth.make_head_case(n_planes=N, tex=R, img=R, n_mpi=1, views_per_mpi=V, seed=11)
    c = dict(rgba=h.rgba.numpy(), view2mpi=h.view2mpi.numpy(), dhw=h.dhw.numpy(), ray_dir=h.ray_dir.numpy(), eye=h.eye.numpy(),
             z_dir=h.z_dir.numpy(), ac=True)
    tau = 2.0 ** -24
    stop = _stop_planes(c, tau)
    tile_stops = []
    for v in range(V):
        for y0 in range(0, R, 30):
            for x0 in range(0, R, 64):
                warps = [int(stop[v, y0 + 2 * w: y0 + 2 * w + 2, x0:x0 + 64].max()) for w in range(15) if y0 + 2 * w < R]
                tile_stops.append(warps)
    assert any(len(set(w)) > 1 and max(w) < N - 1 for w in tile_stops), "no tile whose warps all stop, at different planes"
    assert any(min(w) < N - 1 and max(w) >= N - 1 for w in tile_stops), "no tile where only some warps stop"
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)
    if factored:
        rgb = torch.rand((1, 3, R, R), generator=torch.Generator().manual_seed(12))
        mpi = dict(rgb=t(rgb), alpha=t(c["rgba"][:, :, 3:4]))
        c["rgba"] = g.expand_factored(rgb, torch.from_numpy(c["rgba"][:, :, 3:4].copy())).numpy()
    else:
        mpi = dict(rgba=t(c["rgba"]))
    out = {}
    with forced_kernel(stages):
        for tau_ in (None, 0.0, tau, 0.05):
            with torch.no_grad():
                col, dep = g.render_frames(dhw=t(c["dhw"]), view2mpi=t(c["view2mpi"]), ray_dir=t(c["ray_dir"]), eye=t(c["eye"]),
                                           z_dir=t(c["z_dir"]), view_group=V, early_stop=tau_, **mpi)
            out[tau_] = (col.cpu().numpy(), dep.cpu().numpy())
            if tau_ is not None:
                out[("stats", tau_)] = early_stop_stats()
    assert_bitwise(out[None], out[0.0])
    tiles = -(-R // 64) * -(-R // 30) * V
    assert out[("stats", 0.0)][1] == tiles * N
    for tau_ in (tau, 0.05):      # the producer lags a stopped tile by at most the ring depth; these tiles stop ~N/2 planes early
        skipped, total = out[("stats", tau_)]
        assert total == tiles * N and 0 < skipped < total, (tau_, skipped, total)
    rc, rd, _ = oracle_forward(c)
    for tau_ in (tau, 0.05):
        got = out[tau_]
        for ref in (out[None], (2 * rc - 1, rd)):
            assert np.max(np.abs(got[0] - ref[0])) <= 2 * tau_ + 2 * EXPECT
            excess = np.abs(got[1].astype(np.float64) - ref[1]) - tau_ * max_plane_depth(c) * (1 + 1e-5)
            assert np.max(excess) <= EXPECT * float(np.max(np.abs(ref[1])))


def test_host_entry_point_takes_early_stop():
    """gmpi_mpi_render_host_ex with early_stop renders what the device entry point renders."""
    c = case("small")
    lib = _lib.load()
    V, _, H, W = c["ray_dir"].shape
    M, N = c["rgba"].shape[:2]
    T = c["rgba"].shape[-1]
    h = {k: np.ascontiguousarray(c[k]) for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
    color, depth, flags = np.empty((V, 3, H, W), np.float32), np.empty((V, 1, H, W), np.float32), np.zeros(1, np.uint32)
    d = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | _lib.OPT_EARLY_STOP, early_stop=0.05, M=M, V=V, N=N,
                       Ht=T, Wt=T, H=H, W=W, flags=flags.ctypes.data, color=color.ctypes.data, depth=depth.ctypes.data,
                       **{k: v.ctypes.data for k, v in h.items()})
    _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0))
    dc, dd = render("small", early_stop=0.05)
    assert np.array_equal(color, dc) and np.array_equal(depth, dd)
