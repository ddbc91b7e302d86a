"""LightRenderer mirror (ml_gmpi_b200/light.py, csrc/mpi_light.cuh) against the UNMODIFIED reference's outputs
(tests/golden/light_2x6x32.npz, produced by oracle/make_golden_light.py): compute_depth, the shaded MPI, and both gradients
(through the fused shading kernel, torch's blur / normal ops and the alpha-depth kernel's backward) -- SURVEY.md 8(f) N3."""
import numpy as np
import pytest
import torch

from ml_gmpi_b200.light import LightRenderer, alpha_depth, apply_shading
from ml_gmpi_b200 import expand_factored
from conftest import load_golden, rel_err
from testlib import dev

pytestmark = pytest.mark.gpu


def make_lr():
    lr = LightRenderer(sphere_center_z=1.0, sphere_r=1.0, ka_max=0.7, kd_max=0.6, n_grow_iters=10)
    lr.step = 20
    return lr


def test_compute_depth_and_its_gradient_match_the_reference():
    gd = load_golden("light_2x6x32")
    d = dev()
    t = lambda a: torch.from_numpy(a).to(d)
    alpha = t(gd["mpi"][:, :, 3:]).contiguous().requires_grad_(True)
    depth = alpha_depth(alpha, t(gd["dhw"][:, :1]))
    assert rel_err(depth.detach().cpu().numpy(), gd["depth"]) <= 2e-6
    (depth * t(gd["g_depth"])).sum().backward()
    assert rel_err(alpha.grad.cpu().numpy(), gd["g_alpha_depth"]) <= 5e-6
    # the channel-3 VIEW of an expanded stack is read in place (no copy): same result
    mpi = t(gd["mpi"])
    depth2 = alpha_depth(mpi[:, :, 3:], t(gd["dhw"][:, :1]))
    assert torch.equal(depth2, depth.detach())


def test_render_matches_the_reference_shaded_mpi_and_gradient():
    gd = load_golden("light_2x6x32")
    d = dev()
    t = lambda a: torch.from_numpy(a).to(d)
    lr = make_lr()
    mpi = t(gd["mpi"]).requires_grad_(True)
    out = lr.render(mpi, t(gd["dhw"]), t(gd["xyz"]), given_yaws=torch.from_numpy(gd["light_yaws"]).reshape(-1, 1),
                    given_pitches=torch.from_numpy(gd["light_pitches"]).reshape(-1, 1))
    assert abs(lr.cur_ka - float(gd["ka"])) < 1e-7 and abs(lr.cur_kd - float(gd["kd"])) < 1e-7
    assert out.shape == mpi.shape and rel_err(out.detach().cpu().numpy(), gd["out"]) <= 1e-5
    assert torch.equal(out[:, :, 3], mpi[:, :, 3])                       # alpha untouched (light_renderer.py:197)
    (out * t(gd["g_out"])).sum().backward()
    assert rel_err(mpi.grad.cpu().numpy(), gd["g_mpi"]) <= 5e-5         # through clip mask, normals, blur and the depth composite


def test_seeded_render_draws_the_reference_light():
    """No given light: after torch.manual_seed(5) the mirror consumes the global generator like the reference (blur's sigma draw,
    then the light's truncated normals), so the shaded MPI equals the reference's output for that seed."""
    gd = load_golden("light_2x6x32")
    d = dev()
    t = lambda a: torch.from_numpy(a).to(d)
    lr = make_lr()
    torch.manual_seed(5)
    out = lr.render(t(gd["mpi"]), t(gd["dhw"]), t(gd["xyz"]))
    assert rel_err(out.cpu().numpy(), gd["out"]) <= 1e-5


def test_factored_shading_equals_shading_the_expanded_stack():
    gd = load_golden("light_2x6x32")
    d = dev()
    t = lambda a: torch.from_numpy(a).to(d)
    rgb, alpha = t(gd["mpi"][:, 0, :3]).contiguous(), t(gd["mpi"][:, :, 3:]).contiguous()
    kw = dict(given_yaws=torch.from_numpy(gd["light_yaws"]).reshape(-1, 1), given_pitches=torch.from_numpy(gd["light_pitches"]).reshape(-1, 1))
    shaded_rgb = make_lr().shade_factored(rgb, alpha, t(gd["dhw"]), t(gd["xyz"]), **kw)
    full = make_lr().render(expand_factored(rgb, alpha), t(gd["dhw"]), t(gd["xyz"]), **kw)
    for i in range(alpha.shape[1]):
        assert rel_err(shaded_rgb.cpu().numpy(), full[:, i, :3].cpu().numpy()) <= 1e-6


def test_factored_and_expanded_shading_keep_nan_at_the_same_texels():
    """A NaN colour (a diverging generator) stays NaN through the fused shading, as it does through shade_factored's torch.clip:
    the two paths agree on where the NaNs are and on every other value."""
    gd = load_golden("light_2x6x32")
    d = dev()
    t = lambda a: torch.from_numpy(a).to(d)
    rgb, alpha = t(gd["mpi"][:, 0, :3]).contiguous(), t(gd["mpi"][:, :, 3:]).contiguous()
    rgb[0, 1, 3, 5] = float("nan")
    rgb[1, :, 10, 20] = float("nan")
    rgb[1, 2, 0, 0] = float("inf")
    kw = dict(given_yaws=torch.from_numpy(gd["light_yaws"]).reshape(-1, 1), given_pitches=torch.from_numpy(gd["light_pitches"]).reshape(-1, 1))
    shaded_rgb = make_lr().shade_factored(rgb, alpha, t(gd["dhw"]), t(gd["xyz"]), **kw)
    full = make_lr().render(expand_factored(rgb, alpha), t(gd["dhw"]), t(gd["xyz"]), **kw)
    nan = torch.isnan(shaded_rgb)
    assert int(nan.sum()) == 4
    for i in range(alpha.shape[1]):
        assert torch.equal(torch.isnan(full[:, i, :3]), nan)
        assert rel_err(shaded_rgb[~nan].cpu().numpy(), full[:, i, :3][~nan].cpu().numpy()) <= 1e-6


def test_apply_shading_full_size_stream():
    """One 32-plane 512^2 batch: the fused pass equals the three torch ops it replaces, bit for bit."""
    d = dev()
    gen = torch.Generator(device=d).manual_seed(0)
    mpi = torch.rand((2, 32, 4, 512, 512), generator=gen, device=d)
    shade = torch.rand((2, 1, 512, 512), generator=gen, device=d) * 1.6
    out = apply_shading(mpi, shade)
    ref = torch.cat((torch.clip(mpi[:, :, :3] * shade.unsqueeze(1), min=0.0, max=1.0), mpi[:, :, 3:]), dim=2)
    assert torch.equal(out, ref)
