"""The staged backward's fixed-point gradient box at its limits (run on an H100: pytest -m gpu).

The box kernel adds every (pixel, plane) contribution to a shared-memory int32 box, scaled by a per-tile power of two taken
from the tile's largest upstream gradient (csrc/mpi_bwd_box.cuh).  These tests push that scheme where it cannot hold -- many
pixels per texel (magnification), upstream gradients near the ends of the fp32 range, inf/NaN upstream gradients -- and
compare with the oracle (fp32 autograd formula), through the expanded and the factored backward.  The kernel must then take
its generic body (fp32 global atomics) instead of wrapping or rounding to garbage."""
import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import synth
from conftest import rel_err
from testlib import (EXPECT, FACTORED_RGB_EXPECT, check_factored, dev, expanded_grad, factored_grads, factored_refs, forced_kernel,
                     kernel_fixture, oracle_backward, one_tile_per_mpi_case, upstream)

pytestmark = pytest.mark.gpu
bwd_variant = kernel_fixture("staged", "direct")


@pytest.fixture
def staged():
    """TMA-staged forward and box backward whatever the number of tiles."""
    with forced_kernel("staged"):
        yield


# ------------------------------------------------------------------------------------------------------------------------
# 1. magnification: many pixels per texel within one 64x24 tile
# ------------------------------------------------------------------------------------------------------------------------
def _coherent_mpi(tex, N, d):
    """Plane 0 red with alpha 0.5, black planes behind it, an opaque black last plane: with g_color = (1, 0, 0) every pixel's
    alpha contribution on plane 0 has the same sign and the largest size the tile's scale allows."""
    rgba = torch.zeros((1, N, 4, tex, tex), device=d)
    rgba[0, 0, 0] = 1.0
    rgba[0, 0, 3] = 0.5
    rgba[0, 1:N - 1, 3] = 0.3
    rgba[0, N - 1, 3] = 1.0
    # factored form: red shared colour, black background, the same alphas (the middle planes are red here, not black)
    rgb = torch.zeros((1, 3, tex, tex), device=d)
    rgb[0, 0] = 1.0
    alpha = rgba[:, :, 3:4].clone()
    bg = torch.zeros((1, 3, tex, tex), device=d)
    return rgba, rgb, alpha, bg


@pytest.mark.parametrize("loss", ["red", "color_and_depth"])
@pytest.mark.parametrize("pose", ["identity", "oblique"])
@pytest.mark.parametrize("tex", [256, 64, 32, 16, 8])
def test_magnified_texture_gradient_box_does_not_wrap(tex, pose, loss, staged):
    """Textures of 256^2 down to 8^2 rendered at 512^2 (up to ~60 pixels per texel in each direction)."""
    d = dev()
    N, img = 4, 512
    yaws, pitches = ([0.0], [0.0]) if pose == "identity" else ([0.35], [-0.15])
    case = synth.make_case(n_planes=N, tex=tex, img=img, n_mpi=1, seed=3, device=d, yaws=yaws, pitches=pitches, rgba=False)
    rgba, rgb, alpha, bg = _coherent_mpi(tex, N, d)
    if loss == "red":
        gc = torch.zeros((1, 3, img, img), device=d)
        gc[:, 0] = 1.0
        gd = None
    else:
        gc, gd = torch.ones((1, 3, img, img), device=d), torch.ones((1, 1, img, img), device=d)
    ref = oracle_backward(case, gc, gd, rgba=rgba)
    assert float(np.abs(ref).max()) > 0
    e = rel_err(expanded_grad(rgba, case, gc, gd), ref)
    assert e <= EXPECT, e
    rgba_f = g.expand_factored(rgb, alpha, bg)
    check_factored(factored_grads(rgb, alpha, bg, case, gc, gd), oracle_backward(case, gc, gd, rgba=rgba_f))


# ------------------------------------------------------------------------------------------------------------------------
# 2. the tile exponent tracks the gradient exactly
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("k", [-40, -13, 0, 7, 40])
def test_power_of_two_scaled_upstream_gradient_scales_the_result_bitwise(k, staged):
    d = dev()
    case = one_tile_per_mpi_case(d)
    gc, gd = upstream(2, 24, 64, 4, device=d)
    s = 2.0 ** k
    base = expanded_grad(case.rgba, case, gc, gd)
    scaled = expanded_grad(case.rgba, case, gc * s, gd * s)
    assert np.array_equal(scaled, base * np.float32(s))
    assert rel_err(base, oracle_backward(case, gc, gd)) <= EXPECT
    # factored: per-plane alpha and the background colour get one flush per texel; the shared colour image sums the planes'
    # flushes with fp32 atomics in flusher order, which is exact only up to that order
    gen = torch.Generator(device=d).manual_seed(6)
    rgb, alpha, bg = (torch.rand(sh, generator=gen, device=d) for sh in ((2, 3, 64, 64), (2, 6, 1, 64, 64), (2, 3, 64, 64)))
    # thin planes keep the background visible (T ~ 0.4 in front of it): its gradient is then not a small fraction of the tile's
    # colour scale, where the box's error is bounded relative to that scale rather than to the background gradient itself
    alpha[:, :-1] *= 0.3
    alpha[:, -1] = 1.0
    fb = factored_grads(rgb, alpha, bg, case, gc, gd)
    fs = factored_grads(rgb, alpha, bg, case, gc * s, gd * s)
    assert np.array_equal(fs[1], fb[1] * np.float32(s)) and np.array_equal(fs[2], fb[2] * np.float32(s))
    assert rel_err(fs[0], fb[0] * np.float32(s)) <= 1e-6
    check_factored(fb, oracle_backward(case, gc, gd, rgba=g.expand_factored(rgb, alpha, bg)))


# ------------------------------------------------------------------------------------------------------------------------
# 3. upstream gradients near the ends of the fp32 range
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("scale", [1e-32, 1e-30, 1e27])
def test_extreme_upstream_gradient_magnitudes(scale, staged):
    """1e27: the tile exponent is past 90; 1e-30: the colour quantum at exponent -90 would be 1e-3 of the gradient; 1e-32: the
    scale constants would no longer be normal floats.  The oracle is fp32 too and handles all three."""
    d = dev()
    case = synth.make_case(n_planes=6, tex=128, img=128, n_mpi=2, seed=17, device=d, last_alpha_one=True)
    gc, gd = ((t * scale).to(d) for t in upstream(2, 128, 128, 8))
    ref = oracle_backward(case, gc, gd)
    assert np.isfinite(ref).all() and float(np.abs(ref).max()) > 0
    e = rel_err(expanded_grad(case.rgba, case, gc, gd), ref)
    assert e <= EXPECT, e
    gen = torch.Generator(device=d).manual_seed(9)
    rgb, alpha, bg = (torch.rand(sh, generator=gen, device=d) for sh in ((2, 3, 128, 128), (2, 6, 1, 128, 128), (2, 3, 128, 128)))
    alpha[:, -1] = 1.0
    check_factored(factored_grads(rgb, alpha, bg, case, gc, gd),
                   oracle_backward(case, gc, gd, rgba=g.expand_factored(rgb, alpha, bg)))


# ------------------------------------------------------------------------------------------------------------------------
# 4. inf / NaN upstream gradients
# ------------------------------------------------------------------------------------------------------------------------
def _check_poisoned(ours, ref, variant, tol=EXPECT):
    """Texels the bad pixels do not reach match the oracle.  Under the bad pixels' footprints the staged kernel, like the
    oracle (grid_sampler_2d_backward), adds every in-texture tap, zero-weight taps included, so 0 * NaN poisons exactly the
    oracle's texels.  The direct kernel skips zero-weight taps: there a poisoned oracle texel may stay finite, but no texel may
    be poisoned that the oracle's is not."""
    ours, ref = np.asarray(ours, np.float64), np.asarray(ref, np.float64)
    bad_ref, bad_ours = ~np.isfinite(ref), ~np.isfinite(ours)
    assert bad_ref.any() and bad_ours.any()
    if variant == "staged":
        assert np.array_equal(bad_ours, bad_ref), (int(bad_ours.sum()), int(bad_ref.sum()))
    else:
        assert not np.any(bad_ours & ~bad_ref)
    ok = ~bad_ref & ~bad_ours
    e = rel_err(ours[ok], ref[ok])
    assert e <= tol, e


def test_nan_and_inf_upstream_gradients_propagate_like_autograd(bwd_variant):
    d = dev()
    case = synth.make_case(n_planes=6, tex=128, img=128, n_mpi=1, seed=23, device=d, last_alpha_one=True)
    gc, gd = upstream(1, 128, 128, 10, device=d)
    gc[0, 0, 30, 40] = float("nan")          # backward tile (px0, py0) = (0, 24)
    gd[0, 0, 100, 100] = float("inf")        # backward tile (64, 96)
    ref = oracle_backward(case, gc, gd)
    _check_poisoned(expanded_grad(case.rgba, case, gc, gd), ref, bwd_variant)
    gen = torch.Generator(device=d).manual_seed(11)
    rgb, alpha, bg = (torch.rand(sh, generator=gen, device=d) for sh in ((1, 3, 128, 128), (1, 6, 1, 128, 128), (1, 3, 128, 128)))
    alpha[:, -1] = 1.0
    ours = factored_grads(rgb, alpha, bg, case, gc, gd)
    refs = factored_refs(oracle_backward(case, gc, gd, rgba=g.expand_factored(rgb, alpha, bg)))
    for o, r, tol in zip(ours, refs, (FACTORED_RGB_EXPECT, EXPECT, EXPECT)):
        _check_poisoned(o, r, bwd_variant, tol)
