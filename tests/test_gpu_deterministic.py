"""The deterministic backward on an H100 (pytest -m gpu): bitwise-repeatable and view-order independent gradients, within the
parity bar of the oracle and of the default backward, on the staged box kernel and on the direct kernel, at the edges where the box
kernel takes its generic body, with inf/NaN upstream gradients, accumulating without GMPI_ZERO_GRAD, and through torch's
deterministic switch."""
import ctypes

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from conftest import rel_err
from testlib import (EXPECT, FACTORED_RGB_EXPECT, assert_bitwise, dev, each_alpha, factored_refs, kernel_fixture, oracle_backward,
                     to_np, upstream)

pytestmark = pytest.mark.gpu


variant = kernel_fixture("staged", "direct")     # staged forward + box backward (whatever the number of tiles), or the direct kernels


def _grads(case, gc, gd, *, deterministic, factored=None, align_corners=True, view_group=1, ray=None, order=None):
    """One render + backward; returns the gradients as numpy arrays (expanded: [g_rgba]; factored: [g_rgb, g_alpha, g_bg_rgb]).
    order: a permutation of the views applied to rays, poses and upstream gradients."""
    ray = case.ray_dir if ray is None else ray
    eye, z, v2m = case.eye, case.z_dir, case.view2mpi
    if order is not None:
        ray, eye, z, v2m, gc = ray[order], eye[order], z[order], v2m[order], gc[order]
        gd = None if gd is None else gd[order]
    kw = dict(align_corners=align_corners, view_group=view_group, deterministic=deterministic)
    if factored is None:
        x = case.rgba.clone().requires_grad_(True)
        color, depth = g.render_views(x, case.dhw, v2m, ray, eye, z, **kw)
        leaves = [x]
    else:
        leaves = [t.clone().requires_grad_(True) for t in factored]
        color, depth = g.render_views_factored(leaves[0], leaves[1], case.dhw, v2m, ray, eye, z, bg_rgb=leaves[2], **kw)
    loss = (color * gc).sum() + ((depth * gd).sum() if gd is not None else 0.0)
    loss.backward()
    return [to_np(t.grad) for t in leaves]


def _factored_mpi(M, N, tex, seed, d):
    gen = torch.Generator(device=d).manual_seed(seed)
    rgb, alpha, bg = (torch.rand(sh, generator=gen, device=d) for sh in ((M, 3, tex, tex), (M, N, 1, tex, tex), (M, 3, tex, tex)))
    alpha[:, :-1] *= 0.5
    alpha[:, -1] = 1.0
    return rgb, alpha, bg


def _check_accuracy(ours, default, ref, factored):
    """Within the oracle's bar (2e-5; the factored colour sums N-1 planes' roundings: twice that), and within the same bar of the
    default backward: the deterministic sums add at most 2^(E-k-1) per contribution and one fp32 rounding to the box kernel's
    per-tile fixed point, which the default backward has too (DESIGN.md section 4.3)."""
    refs = factored_refs(ref) if factored else [ref]
    tols = (FACTORED_RGB_EXPECT, EXPECT, EXPECT) if factored else (EXPECT,)
    for o, d_, r, tol in zip(ours, default, refs, tols):
        assert rel_err(o, r) <= tol, rel_err(o, r)
        assert rel_err(o, d_) <= tol, rel_err(o, d_)


# ------------------------------------------------------------------------------------------------------------------------
# repeatability and accuracy
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("align_corners", [True, False])
@pytest.mark.parametrize("depth", [True, False])
@pytest.mark.parametrize("form", ["expanded", "factored"])
def test_repeatable_and_accurate(form, depth, align_corners, variant):
    d = dev()
    M, vpm, N, tex, img = 2, 2, 12, 128, 256
    case = synth.make_case(n_planes=N, tex=tex, img=img, n_mpi=M, views_per_mpi=vpm, seed=31, device=d, last_alpha_one=True)
    gc, gd = upstream(M * vpm, img, img, 5, depth, d)
    fac = _factored_mpi(M, N, tex, 7, d) if form == "factored" else None
    kw = dict(factored=fac, align_corners=align_corners, view_group=vpm)
    a = _grads(case, gc, gd, deterministic=True, **kw)
    b = _grads(case, gc, gd, deterministic=True, **kw)
    assert_bitwise(a, b)
    rgba = case.rgba if fac is None else g.expand_factored(*fac)
    ref = oracle_backward(case, gc, gd, rgba=rgba, align_corners=align_corners)
    _check_accuracy(a, _grads(case, gc, gd, deterministic=False, **kw), ref, fac is not None)


@pytest.mark.parametrize("form", ["expanded", "factored"])
def test_view_order_does_not_change_a_bit(form, variant):
    """Views of each MPI permuted together with their rays, poses and upstream gradients (and the MPIs' blocks swapped)."""
    d = dev()
    M, vpm, N, tex, img = 2, 3, 8, 128, 192
    case = synth.make_case(n_planes=N, tex=tex, img=img, n_mpi=M, views_per_mpi=vpm, seed=41, device=d, last_alpha_one=True)
    gc, gd = upstream(M * vpm, img, img, 6, device=d)
    fac = _factored_mpi(M, N, tex, 8, d) if form == "factored" else None
    base = _grads(case, gc, gd, deterministic=True, factored=fac)
    for order in ([2, 0, 1, 5, 3, 4], [4, 5, 3, 1, 2, 0]):
        assert_bitwise(base, _grads(case, gc, gd, deterministic=True, factored=fac, order=torch.tensor(order, device=d)))


@each_alpha("variant", ["staged", "direct"], indirect=["variant"])
def test_full_size_training_shape_is_repeatable(variant, alpha):
    """4 MPIs x 1 view, 96 planes, 1024^2 texture and image (12.9 GB of sums: MPIs 2 and 3 start past 2^31 bytes of the gradient,
    their sums past 2^32); every MPI's gradient (its one view's) against the oracle, on its own scale.  With equal-weight alpha every
    plane's gradient is far from 0, so repeatability is not met trivially on the back planes."""
    d = dev()
    case = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=3, device=d, last_alpha_one=True, alpha=alpha)
    gc, gd = upstream(4, 1024, 1024, 9, device=d)
    a = _grads(case, gc, gd, deterministic=True)
    assert_bitwise(a, _grads(case, gc, gd, deterministic=True))
    e = rel_err(a[0], _grads(case, gc, gd, deterministic=False)[0])
    assert e <= EXPECT, e
    ref = oracle_backward(case, gc, gd)
    errs = [rel_err(a[0][m], ref[m]) for m in range(4)]
    assert max(errs) <= EXPECT, errs


def test_fifteen_views_of_one_mpi_are_repeatable(variant):
    """The C4 shape: 15 views of one 96 x 512^2 MPI, all adding into the same gradient."""
    d = dev()
    case = synth.make_case(n_planes=96, tex=512, img=512, n_mpi=1, views_per_mpi=15, seed=4, device=d, last_alpha_one=True)
    gc, gd = upstream(15, 512, 512, 10, device=d)
    a = _grads(case, gc, gd, deterministic=True, view_group=15)
    assert_bitwise(a, _grads(case, gc, gd, deterministic=True, view_group=15))
    e = rel_err(a[0], _grads(case, gc, gd, deterministic=False, view_group=15)[0])
    assert e <= EXPECT, e


# ------------------------------------------------------------------------------------------------------------------------
# where the box kernel takes its generic body (tests/test_gpu_bwd_limits.py)
# ------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tex", [16, 64])
def test_magnified_texture(tex, variant):
    d = dev()
    N, img = 4, 512
    case = synth.make_case(n_planes=N, tex=tex, img=img, n_mpi=1, seed=3, device=d, yaws=[0.35], pitches=[-0.15], last_alpha_one=True)
    gc, gd = torch.ones((1, 3, img, img), device=d), torch.ones((1, 1, img, img), device=d)
    a = _grads(case, gc, gd, deterministic=True)
    assert_bitwise(a, _grads(case, gc, gd, deterministic=True))
    _check_accuracy(a, _grads(case, gc, gd, deterministic=False), oracle_backward(case, gc, gd), False)
    fac = _factored_mpi(1, N, tex, 12, d)
    a = _grads(case, gc, gd, deterministic=True, factored=fac)
    assert_bitwise(a, _grads(case, gc, gd, deterministic=True, factored=fac))
    ref = oracle_backward(case, gc, gd, rgba=g.expand_factored(*fac))
    _check_accuracy(a, _grads(case, gc, gd, deterministic=False, factored=fac), ref, True)


@pytest.mark.parametrize("scale", [1e-32, 1e-30, 1e27])
def test_extreme_upstream_gradient_magnitudes(scale, variant):
    d = dev()
    case = synth.make_case(n_planes=6, tex=128, img=128, n_mpi=2, seed=17, device=d, last_alpha_one=True)
    gc, gd = ((t * scale).to(d) for t in upstream(2, 128, 128, 8))
    a = _grads(case, gc, gd, deterministic=True)
    assert_bitwise(a, _grads(case, gc, gd, deterministic=True))
    ref = oracle_backward(case, gc, gd)
    assert np.isfinite(ref).all() and float(np.abs(ref).max()) > 0
    _check_accuracy(a, _grads(case, gc, gd, deterministic=False), ref, False)
    fac = _factored_mpi(2, 6, 128, 9, d)
    a = _grads(case, gc, gd, deterministic=True, factored=fac)
    assert_bitwise(a, _grads(case, gc, gd, deterministic=True, factored=fac))
    ref = oracle_backward(case, gc, gd, rgba=g.expand_factored(*fac))
    _check_accuracy(a, _grads(case, gc, gd, deterministic=False, factored=fac), ref, True)


# ------------------------------------------------------------------------------------------------------------------------
# inf / NaN upstream gradients
# ------------------------------------------------------------------------------------------------------------------------
def test_non_finite_upstream_gradients(variant):
    """The non-finite pattern (+inf, -inf, NaN per element) equals the default backward's on the same kernel; every other element
    is finite, repeatable, and within the bar of the default backward."""
    d = dev()
    case = synth.make_case(n_planes=6, tex=128, img=128, n_mpi=1, seed=23, device=d, last_alpha_one=True)
    gc, gd = upstream(1, 128, 128, 10, device=d)
    gc[0, 0, 30, 40] = float("nan")
    gd[0, 0, 100, 100] = float("inf")
    gc[0, 1, 70, 20] = float("-inf")
    fac = _factored_mpi(1, 6, 128, 11, d)
    for f in (None, fac):
        a = _grads(case, gc, gd, deterministic=True, factored=f)
        b = _grads(case, gc, gd, deterministic=True, factored=f)
        ref = _grads(case, gc, gd, deterministic=False, factored=f)
        for x, y, r in zip(a, b, ref):
            assert_bitwise(x, y)
            bad = ~np.isfinite(r)
            assert bad.any()
            for kind in (np.isnan, np.isposinf, np.isneginf):
                assert np.array_equal(kind(x), kind(r)), kind.__name__
            assert rel_err(x[~bad], r[~bad]) <= 2 * EXPECT


# ------------------------------------------------------------------------------------------------------------------------
# the C ABI: accumulate without GMPI_ZERO_GRAD
# ------------------------------------------------------------------------------------------------------------------------
def test_accumulates_without_zero_grad(variant):
    d = dev()
    lib = _lib.load()
    case = synth.make_case(n_planes=8, tex=128, img=256, n_mpi=2, views_per_mpi=2, seed=51, device=d, last_alpha_one=True)
    M, N, V, H, W = 2, 8, 4, 256, 256
    gc, gd = upstream(V, H, W, 12, device=d)
    color, depth = torch.empty((V, 3, H, W), device=d), torch.empty((V, 1, H, W), device=d)
    trans = torch.empty((V, N, H, W), device=d)
    flags = torch.zeros(1, dtype=torch.int32, device=d)
    common = dict(M=M, V=V, N=N, Ht=128, Wt=128, H=H, W=W, view_group=2, rgba=case.rgba, view2mpi=case.view2mpi, dhw=case.dhw,
                  ray_dir=case.ray_dir, eye=case.eye, z_dir=case.z_dir, transmittance=trans, stream=torch.cuda.current_stream().cuda_stream)
    _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(_lib.make_desc(options=_lib.OPT_ALIGN_CORNERS, color=color, depth=depth,
                                                                        flags=flags, **common))))

    def bwd(g_rgba, options):
        desc = _lib.make_desc(options=options, g_color=gc, g_depth=gd, g_rgba=g_rgba, **common)
        nbytes = _lib.deterministic_scratch_bytes(desc)
        scratch = torch.empty(nbytes, dtype=torch.uint8, device=d)
        _lib.check(lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(desc), scratch.data_ptr(), nbytes))
        return g_rgba

    fresh = to_np(bwd(torch.full_like(case.rgba, float("nan")), _lib.OPT_ALIGN_CORNERS | _lib.OPT_ZERO_GRAD))
    prefill = torch.randn(case.rgba.shape, generator=torch.Generator().manual_seed(13)).to(d)
    added = to_np(bwd(prefill.clone(), _lib.OPT_ALIGN_CORNERS))
    assert np.isfinite(fresh).all()
    assert np.array_equal(added, to_np(prefill) + fresh)


# ------------------------------------------------------------------------------------------------------------------------
# through torch
# ------------------------------------------------------------------------------------------------------------------------
def _train_step(case, gc, gd, mpi):
    x = case.rgba.clone().requires_grad_(True)
    v2m = to_np(case.view2mpi)
    idx = [np.nonzero(v2m == m)[0] for m in range(case.rgba.shape[0])]
    color, depth = mpi(batch_rgba=x, batch_dhw=case.dhw, batch_ray_dir=[case.ray_dir[i] for i in idx],
                       batch_eye_pos=[case.eye[i] for i in idx], batch_z_dir=[case.z_dir[i] for i in idx], separate_background=None)
    ((color * gc).sum() + (depth * gd).sum()).backward()
    return to_np(x.grad)


def test_torch_deterministic_switch_selects_the_deterministic_backward(monkeypatch):
    d = dev()
    lib = _lib.load()
    calls = []
    real = lib.gmpi_mpi_render_bwd_deterministic_ex

    def spy(*args):
        calls.append(1)
        return real(*args)

    monkeypatch.setattr(lib, "gmpi_mpi_render_bwd_deterministic_ex", spy)
    case = synth.make_case(n_planes=16, tex=256, img=256, n_mpi=2, views_per_mpi=2, seed=61, device=d, last_alpha_one=True)
    gc, gd = upstream(4, 256, 256, 14, device=d)
    mpi = g.MPI(align_corners=True, validate="full")
    default = _train_step(case, gc, gd, mpi)
    assert calls == []
    was = torch.are_deterministic_algorithms_enabled()
    torch.use_deterministic_algorithms(True)
    try:
        a = _train_step(case, gc, gd, mpi)
        b = _train_step(case, gc, gd, mpi)
    finally:
        torch.use_deterministic_algorithms(was)
    assert len(calls) == 2
    assert_bitwise([a], [b])
    assert rel_err(a, default) <= EXPECT
    # the constructor's option overrides the switch, in both directions
    _train_step(case, gc, gd, g.MPI(align_corners=True, deterministic=True))
    assert len(calls) == 3
    torch.use_deterministic_algorithms(True)
    try:
        _train_step(case, gc, gd, g.MPI(align_corners=True, deterministic=False))
    finally:
        torch.use_deterministic_algorithms(was)
    assert len(calls) == 3
