"""The factored MPI (shared colour rgb [M,3,Ht,Wt], optional bg_rgb for the last plane, per-plane alpha [M,N,1,Ht,Wt]) against the
oracle on the expanded stack, on the direct kernels and on the TMA-staged forward + box backward (run on an H100: pytest -m gpu).

The factored kernels are template instantiations of their own (mpi_fwd_staged_kernel<kKeyFac | ...>, mpi_bwd_box_kernel<kKeyFac | ...>) with
their own ring and box layout, so every edge the expanded kernels are tested at (tests/testlib.py's case catalogue) is repeated here:
align_corners=False, non-square textures, partial tiles, N = 1 and N = 512, footprints 89..96 texels wide (they fit the factored forward's 96-wide box but take the
generic body, as in the expanded ring) and wider than 96, non-pinhole and degenerate rays, MPIs without views, views in any order, GMPI_ZERO_GRAD, view_group, unaligned
factors, the host entry point and the benchmark's own shapes.

Reference: mpi_oracle on expand_factored(rgb, alpha, bg_rgb): colour and depth; d alpha = the oracle's g_rgba[:, :, 3];
d rgb = the sum of g_rgba[:, :last, :3] over planes, in float64 (last = N - 1 with bg_rgb, else N); d bg_rgb = g_rgba[:, -1, :3].

Bars (derived, not fitted):
  forward      bitwise the expanded render on the same kernel (DESIGN.md, N1), and rel_err <= EXPECT against the oracle for
               colour and depth (EXPECT: the expanded kernels' bar, tests/testlib.py).
  d alpha      rel_err <= EXPECT: the alpha box is the expanded path's 26-bit fixed point, one plane per texel.
  d rgb, d bg  max|ours - ref| / S, S = max|oracle g_rgba| over all planes and channels.  The box backward rounds every colour
               contribution to a multiple of 2^(e_rgb - kFixBitsRgb) (kFixBitsRgb = 22, csrc/mpi_bwd_box.cuh) with 2^e_rgb <= 4 gmax
               (tile_scale_exponent(gmax / 2); gmax = the largest |upstream colour gradient| the kernel sees, x2 under
               color_minus1_1), i.e. by at most 2^(e_rgb - 23) <= 2^-21 gmax.  A texel of d rgb sums K such contributions: every
               bilinear tap of every pixel of every view of its MPI on each of the planes that share rgb (up to N - 1 of them), so
                   max|ours - ref| <= K * 2^-21 * gmax + (fp32 accumulation, ours and the oracle's)
               and the bar is  K * 2^-21 * gmax / S + EXPECT,  with K counted exactly per case from the texel coordinates
               (_tap_counts; zero-weight taps are counted too, which only loosens it).  d bg_rgb: the same with the last plane's K.
               This is relative to the tile's gradient scale, not to the factor: behind near-opaque planes d bg is tiny and its own
               relative error is not small even when the kernel is right (test_gpu_bwd_limits.py, section 2).
  d bg visible where the background is built to show (transmittance in front of the last plane mostly >= 0.1: the other alphas
               scaled down), also rel_err(d bg) <= EXPECT against its own maximum: the S-normalised bar alone would accept a kernel
               that sent the background's gradient to d rgb.
test_the_bars_fail_on_a_slightly_wrong_problem shows that these bars fail by 10x or more on slightly wrong problems."""
import ctypes
import functools
import json

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib
from conftest import MPI_CASES, rel_err
from testlib import (EXPECT, GEOMETRY, assert_bitwise, case, dev, expanded_grad, factored_grads, forced_kernel, kernel_fixture,
                     limit_footprints, misaligned, on_device, one_tile_per_mpi_case, oracle_backward, oracle_forward, pixels, to_np,
                     upstream)

pytestmark = pytest.mark.gpu
FIX_BITS_RGB = 22                  # kFixBitsRgb, csrc/mpi_bwd_box.cuh
ROUND_RGB = 2.0 ** -(FIX_BITS_RGB - 1)   # largest rounding of one colour contribution, in units of gmax: 2^(e_rgb - 23) / gmax


# The direct kernels, or the staged forward + box backward forced whatever the number of tiles (the factored ring is always 3 deep:
# the ring depth does not apply to it).
variant = kernel_fixture("direct", "staged")


# the catalogue's cases (tests/testlib.py): geometry, factors and upstream gradients
GOLDEN = MPI_CASES + ["edge_odd_sizes", "edge_single_plane", "edge_acfalse_nonsquare", "edge_ragged_zero_views"]
MATRIX = GOLDEN + ["partial_acfalse_nonsquare", "N1", "N512", "band_89_96", "wider_than_96", "shuffled_rays", "corners_off_the_planes",
                   "degenerate_rays", "bench_96x1024", "views4_48x512", "bench_96x1024_equal_weight", "views4_48x512_equal_weight"]


def _mpi(c, with_bg):
    """The factored MPI (rgb, alpha, bg_rgb or None) of case c on the device."""
    rgb, alpha, bg = on_device(c, "rgb", "alpha", "bg")
    return rgb, alpha, bg if with_bg else None


def _expand(c, with_bg):
    t = torch.from_numpy
    return g.expand_factored(t(c["rgb"]), t(c["alpha"]), t(c["bg"]) if with_bg else None).numpy()


# ------------------------------------------------------------------------------------------------------------------------------
# the reference, once per case and session; only what the checks need is kept (the expanded stacks of the large cases are not)
# ------------------------------------------------------------------------------------------------------------------------------
WRONG = ["last_plane_from_rgb", "rgb_shifted_one_column", "align_corners_flipped", "views_of_two_mpis_swapped"]


@functools.lru_cache(maxsize=None)
def reference(name, with_bg, wrong=None):
    """Oracle of the case, or of a slightly wrong version of it (WRONG): the bars must fail on those."""
    c = dict(case(name))
    expand_bg = with_bg and wrong != "last_plane_from_rgb"
    if wrong == "rgb_shifted_one_column":
        c["rgb"] = np.roll(c["rgb"], 1, axis=-1)
    if wrong == "align_corners_flipped":
        c["ac"] = not c["ac"]
    if wrong == "views_of_two_mpis_swapped":
        v2m = c["view2mpi"].copy()
        c["view2mpi"] = np.where(v2m == 0, 1, np.where(v2m == 1, 0, v2m)).astype(np.int32)
    rgba = _expand(c, expand_bg)
    color, depth, flags = oracle_forward(c, rgba=rgba, align_corners=c["ac"], check_last_plane=True)
    gc = c["gc"] * (2.0 if c.get("m11") else 1.0)         # the kernel's upstream gradient w.r.t. c when the output is 2c - 1
    G = oracle_backward(c, gc, c["gd"], rgba=rgba, align_corners=c["ac"])
    del rgba
    N = G.shape[1]
    last = N - 1 if with_bg else N
    return dict(color=2 * color - 1 if c.get("m11") else color, depth=depth, flags=flags, g_rgb=G[:, :last, :3].astype(np.float64).sum(1),
                g_alpha=G[:, :, 3:4].copy(), g_bg=G[:, -1, :3].copy() if with_bg else None, S=float(np.abs(G).max()),
                gmax=float(np.abs(gc).max()))


@functools.lru_cache(maxsize=None)
def _tap_counts(name):
    """(K of the planes in front of the last, K of the last plane, K of all planes): the largest number of bilinear taps any texel
    receives, over all views of its MPI, from the pixels' texel coordinates (gmpi_debug_plane_coords, bit-exact with the oracle's)."""
    c = case(name)
    d = dev()
    lib = _lib.load()
    dhws, rays, eyes = on_device(c, "dhw", "ray_dir", "eye")
    M, N, _, Ht, Wt = c["alpha"].shape
    V, _, H, W = c["ray_dir"].shape
    front, last = torch.zeros((M, Ht * Wt), dtype=torch.int64, device=d), torch.zeros((M, Ht * Wt), dtype=torch.int64, device=d)
    zero = torch.zeros(1, dtype=torch.int32, device=d)
    out = torch.empty((1, 1, 2, H, W), device=d)
    for v in range(V):
        m = int(c["view2mpi"][v])
        ray, eye = rays[v:v + 1], eyes[v:v + 1]
        for i in range(N):
            dhw = dhws[m:m + 1, i:i + 1]
            _lib.check(lib.gmpi_debug_plane_coords(zero.data_ptr(), dhw.data_ptr(), ray.data_ptr(), eye.data_ptr(), out.data_ptr(),
                                                    1, 1, Ht, Wt, H, W, _lib.OPT_ALIGN_CORNERS if c["ac"] else 0, None))
            ix, iy = out[0, 0, 0].flatten(), out[0, 0, 1].flatten()
            ok = torch.isfinite(ix) & torch.isfinite(iy)
            x0 = ix[ok].clamp(-2, Wt + 1).floor().long()
            y0 = iy[ok].clamp(-2, Ht + 1).floor().long()
            hist = front[m] if i < N - 1 else last[m]
            for dy in (0, 1):
                for dx in (0, 1):
                    x, y = x0 + dx, y0 + dy
                    inside = (x >= 0) & (x < Wt) & (y >= 0) & (y < Ht)
                    hist += torch.bincount((y * Wt + x)[inside], minlength=Ht * Wt)
    return int(front.max()), int(last.max()), int((front + last).max())


def bars(name, with_bg, ref):
    kf, kl, ka = _tap_counts(name)
    k_rgb = kf if with_bg else ka
    b = dict(color=EXPECT, depth=EXPECT, g_alpha=EXPECT, g_rgb=k_rgb * ROUND_RGB * ref["gmax"] / ref["S"] + EXPECT)
    if with_bg:
        b["g_bg"] = kl * ROUND_RGB * ref["gmax"] / ref["S"] + EXPECT
        if case(name).get("visible"):
            b["g_bg_own"] = EXPECT
    return b


def errors(ours, ref, c):
    """The measured figure of every check (compare with bars())."""
    S = ref["S"]
    e = dict(color=rel_err(pixels(c, ours["color"]), pixels(c, ref["color"])), depth=rel_err(pixels(c, ours["depth"]), pixels(c, ref["depth"])),
             g_alpha=rel_err(ours["g_alpha"], ref["g_alpha"]),
             g_rgb=float(np.max(np.abs(ours["g_rgb"].astype(np.float64) - ref["g_rgb"]))) / S)
    if ref["g_bg"] is not None:
        e["g_bg"] = float(np.max(np.abs(ours["g_bg"].astype(np.float64) - ref["g_bg"]))) / S
        if c.get("visible"):
            e["g_bg_own"] = rel_err(ours["g_bg"], ref["g_bg"])
    return e


def check(label, ours, name, with_bg, plan_=None):
    ref = reference(name, with_bg)
    c = case(name)
    e, b = errors(ours, ref, c), bars(name, with_bg, ref)
    print("FACTORED " + json.dumps(dict(case=label, plan=plan_, err={k: float("%.3g" % v) for k, v in e.items()},
                                        bar={k: float("%.3g" % v) for k, v in b.items()})))
    assert np.isfinite(ours["g_rgb"]).all() and np.isfinite(ours["g_alpha"]).all()
    bad = {k: (e[k], b[k]) for k in b if not e[k] <= b[k]}
    assert not bad, (label, bad)
    if "flags" in ours:
        assert ours["flags"] == ref["flags"], (label, ours["flags"], ref["flags"])


# ------------------------------------------------------------------------------------------------------------------------------
# running the factored render
# ------------------------------------------------------------------------------------------------------------------------------
def fwd_plan(c, mpi, view_group=1):
    V, _, H, W = c["ray_dir"].shape
    M, N, _, Ht, Wt = c["alpha"].shape
    desc = _lib.make_desc(options=0, M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, view_group=view_group, rgb=mpi[0], alpha=mpi[1], bg_rgb=mpi[2])
    p, why = _lib.fwd_plan(desc)
    return ("staged" if p == _lib.PLAN_STAGED else "direct"), why


def run(name, with_bg, mpi=None, view_group=1):
    """render_views_factored forward-only and with autograd, each bitwise against the expanded render on the same kernel, then the
    backward.  mpi: (rgb, alpha, bg_rgb) device tensors to render instead of the case's (their storage is kept)."""
    c = case(name)
    d = dev()
    base, geo = _mpi(c, with_bg), on_device(c, *GEOMETRY)
    mpi = base if mpi is None else mpi
    kw = dict(align_corners=c["ac"], check_last_plane=True, color_minus1_1=c.get("m11", False), view_group=view_group)
    flags = lambda: torch.zeros(1, dtype=torch.int32, device=d)
    x = g.expand_factored(*base)
    if any(t is not None and t.data_ptr() % 16 for t in mpi):
        x = misaligned(x, 4)                # the expanded stack takes the direct kernel too
    with torch.no_grad():
        ff, fe = flags(), flags()
        cf, df = g.render_views_factored(mpi[0], mpi[1], *geo, bg_rgb=mpi[2], flags=ff, **kw)
        ce, de = g.render_views(x, *geo, flags=fe, **kw)
    assert_bitwise((cf, df), (ce, de), (name, "forward-only kernel != expanded"))
    assert int(ff.item()) == int(fe.item())
    leaves = [None if v is None else v.detach().requires_grad_(True) for v in mpi]
    xe = x.detach().requires_grad_(True)
    ft, fte = flags(), flags()
    col, dep = g.render_views_factored(leaves[0], leaves[1], *geo, bg_rgb=leaves[2], flags=ft, **kw)
    ce2, de2 = g.render_views(xe, *geo, flags=fte, **kw)
    assert_bitwise((col, dep), (ce2, de2), (name, "training forward != expanded"))
    assert_bitwise((col, dep), (cf, df), (name, "training forward != forward-only kernel"))
    del ce2, de2, xe, x
    gc, gd = on_device(c, "gc", "gd")
    loss = (col * gc).sum()
    if gd is not None:
        loss = loss + (dep * gd).sum()
    loss.backward()
    out = dict(color=to_np(col), depth=to_np(dep), flags=int(ft.item()), g_rgb=to_np(leaves[0].grad), g_alpha=to_np(leaves[1].grad),
               g_bg=to_np(leaves[2].grad) if with_bg else None)
    assert int(ff.item()) == out["flags"]
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# 1. the matrix
# ------------------------------------------------------------------------------------------------------------------------------
# with and without bg_rgb, except at the two operating points: the benchmark renders without one, the four-view case with one
_BGS = {"bench_96x1024": (False,), "views4_48x512": (True,), "bench_96x1024_equal_weight": (False,), "views4_48x512_equal_weight": (True,)}


def _matrix_params():
    for name in MATRIX:
        for bg in _BGS.get(name, (False, True)):
            yield pytest.param(name, bg, id=f"{name}-{'bg' if bg else 'nobg'}")


@pytest.mark.parametrize("name,with_bg", list(_matrix_params()))
def test_factored_matches_the_oracle(name, with_bg, variant):
    c = case(name)
    mpi = _mpi(c, with_bg)
    Wt = c["alpha"].shape[-1]
    p, why = fwd_plan(c, mpi)
    if variant == "direct":
        assert p == "direct"
    elif Wt % 4:
        assert (p, why) == ("direct", 1)           # Wt % 4 != 0: no tensor map, the direct kernel whatever is forced
    else:
        assert p == "staged", why
    if name == "band_89_96":
        assert limit_footprints(c, 89, 96) > 0
    if name == "wider_than_96":
        assert limit_footprints(c, 97, 1 << 30) > 0
    ours = run(name, with_bg)
    if name == "N1" and with_bg:
        assert not ours["g_rgb"].any()              # the one plane is the background: nothing reaches rgb
    check(f"{name}/{'bg' if with_bg else 'nobg'}/{variant}", ours, name, with_bg, p)


# ------------------------------------------------------------------------------------------------------------------------------
# 2. one integer flush per texel and plane: the factored box backward is bitwise the expanded one
# ------------------------------------------------------------------------------------------------------------------------------
def test_one_tile_per_mpi_factored_gradients_are_bitwise_the_expanded_ones():
    """testlib.one_tile_per_mpi_case: every texel gets exactly one integer flush per plane, so d alpha and d bg of the
    staged factored backward equal the expanded backward's g_rgba[:, :, 3] and g_rgba[:, -1, :3] bit for bit."""
    d = dev()
    with forced_kernel("staged"):
        geo = one_tile_per_mpi_case(d)
        gc, gd = upstream(2, 24, 64, 4, device=d)
        gen = torch.Generator(device=d).manual_seed(6)
        rgb, alpha, bg = (torch.rand(sh, generator=gen, device=d) for sh in ((2, 3, 64, 64), (2, 6, 1, 64, 64), (2, 3, 64, 64)))
        alpha[:, :-1] *= 0.3
        alpha[:, -1] = 1.0
        f_rgb, f_alpha, f_bg = factored_grads(rgb, alpha, bg, geo, gc, gd)
        e = expanded_grad(g.expand_factored(rgb, alpha, bg), geo, gc, gd)
    assert_bitwise(f_alpha[:, :, 0], e[:, :, 3], "d alpha")
    assert_bitwise(f_bg, e[:, -1, :3], "d bg_rgb")
    assert rel_err(f_rgb, e[:, :-1, :3].astype(np.float64).sum(1)) <= 1e-6         # fp32 atomics over the planes: order only


# ------------------------------------------------------------------------------------------------------------------------------
# 3. through the C ABI: view order, GMPI_ZERO_GRAD into NaN, accumulation, MPIs without views
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ["sorted", "interleaved", "reversed"])
def test_zero_grad_poisoned_buffers_any_view_order(order, variant):
    name = "three_mpis_" + order
    c = case(name)
    d = dev()
    lib = _lib.load()
    (rgb, alpha, bg), (dhw, v2m, ray, eye, z) = _mpi(c, True), on_device(c, *GEOMETRY)
    M, N, _, Ht, Wt = alpha.shape
    V, _, H, W = ray.shape
    opt = _lib.OPT_ALIGN_CORNERS | _lib.OPT_CHECK_LAST_PLANE
    color, depth = torch.empty((V, 3, H, W), device=d), torch.empty((V, 1, H, W), device=d)
    trans = torch.empty((V, N, H, W), device=d)
    flags = torch.zeros(1, dtype=torch.int32, device=d)
    common = dict(M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, rgb=rgb, alpha=alpha, bg_rgb=bg, view2mpi=v2m, dhw=dhw, ray_dir=ray, eye=eye,
                  z_dir=z, stream=torch.cuda.current_stream(d).cuda_stream)
    _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(_lib.make_desc(options=opt, color=color, depth=depth, transmittance=trans,
                                                                      flags=flags, **common))))
    gc, gd = on_device(c, "gc", "gd")

    def bwd(fill, options):
        gr, ga, gb = torch.full_like(rgb, fill), torch.full_like(alpha, fill), torch.full_like(bg, fill)
        _lib.check(lib.gmpi_mpi_render_bwd_ex(ctypes.byref(_lib.make_desc(options=options, transmittance=trans, g_color=gc, g_depth=gd,
                                                                          g_rgb=gr, g_alpha=ga, g_bg_rgb=gb, **common))))
        torch.cuda.synchronize()
        return [t.cpu().numpy() for t in (gr, ga, gb)]

    out = dict(color=to_np(color), depth=to_np(depth), flags=int(flags.item()))
    z_rgb, z_alpha, z_bg = bwd(float("nan"), opt | _lib.OPT_ZERO_GRAD)
    assert not (z_rgb[3].any() or z_alpha[3].any() or z_bg[3].any()), "an MPI without views must get exactly 0"
    check(f"{name}/zero_grad/{variant}", dict(out, g_rgb=z_rgb, g_alpha=z_alpha, g_bg=z_bg), name, True)
    a_rgb, a_alpha, a_bg = bwd(1.0, opt)
    assert (a_rgb[3] == 1).all() and (a_alpha[3] == 1).all() and (a_bg[3] == 1).all(), "an MPI without views: buffer untouched"
    check(f"{name}/accumulate/{variant}", dict(g_rgb=a_rgb - 1.0, g_alpha=a_alpha - 1.0, g_bg=a_bg - 1.0, color=out["color"],
                                                depth=out["depth"]), name, True)


# ------------------------------------------------------------------------------------------------------------------------------
# 4. view_group, unaligned factors, the host entry point
# ------------------------------------------------------------------------------------------------------------------------------
def test_view_group_changes_no_output_bit_and_no_gradient_beyond_the_bar(variant):
    name = "view_group"
    outs = {vg: run(name, True, view_group=vg) for vg in (1, 2, 4)}
    ref = reference(name, True)
    for vg, o in outs.items():
        for k in ("color", "depth"):
            assert_bitwise(o[k], outs[1][k], (vg, k))
        check(f"{name}/view_group={vg}/{variant}", o, name, True)
        # and against view_group = 1 with the same bars (the group-1 result as the reference)
        one = dict(ref, **{k: outs[1][k] for k in ("color", "depth", "g_alpha", "g_bg")},
                   g_rgb=outs[1]["g_rgb"].astype(np.float64))
        e, b = errors(o, one, case(name)), bars(name, True, ref)
        assert all(e[k] <= b[k] for k in b), (vg, e, b)


@pytest.mark.parametrize("which", ["rgb", "alpha", "bg_rgb"])
def test_one_unaligned_factor_takes_the_direct_kernels(which, variant):
    name = "small_12x96"
    c = case(name)
    mpi = _mpi(c, True)
    i = ["rgb", "alpha", "bg_rgb"].index(which)
    mpi = tuple(misaligned(t, 4) if j == i else t for j, t in enumerate(mpi))
    p, why = fwd_plan(c, mpi)
    assert p == "direct" and why & 8, (p, why)
    check(f"{name}/unaligned_{which}/{variant}", run(name, True, mpi=mpi), name, True, p)


@pytest.mark.parametrize("with_bg", [False, True])
def test_host_entry_point_with_ray_tensors_is_bitwise_the_device_call(with_bg, variant):
    name = "small_12x96"
    c = case(name)
    d = dev()
    lib = _lib.load()
    M, N, _, Ht, Wt = c["alpha"].shape
    V, _, H, W = c["ray_dir"].shape
    opt = _lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | _lib.OPT_CHECK_LAST_PLANE
    sizes = dict(options=opt, M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W)
    keys = ("rgb", "alpha", "view2mpi", "dhw", "ray_dir", "eye", "z_dir") + (("bg",) if with_bg else ())
    h = {k: np.ascontiguousarray(c[k]) for k in keys}
    color, depth, flags = np.empty((V, 3, H, W), np.float32), np.empty((V, 1, H, W), np.float32), np.zeros(1, np.uint32)
    ptr = {("bg_rgb" if k == "bg" else k): v.ctypes.data for k, v in h.items()}
    _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(_lib.make_desc(color=color.ctypes.data, depth=depth.ctypes.data,
                                                                       flags=flags.ctypes.data, **sizes, **ptr)), 0))
    t = {("bg_rgb" if k == "bg" else k): torch.from_numpy(v).to(d) for k, v in h.items()}
    dc, dd = torch.empty((V, 3, H, W), device=d), torch.empty((V, 1, H, W), device=d)
    df = torch.zeros(1, dtype=torch.int32, device=d)
    _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(_lib.make_desc(color=dc, depth=dd, flags=df, **sizes, **t))))
    torch.cuda.synchronize()
    assert_bitwise((color, depth), (dc, dd), "host entry point != device entry point")
    assert int(flags[0]) == int(df.item())
    ref = reference(name, with_bg)
    assert rel_err(color, 2 * ref["color"] - 1) <= EXPECT and rel_err(depth, ref["depth"]) <= EXPECT
    _lib.check(lib.gmpi_mpi_release_host_cache())


# ------------------------------------------------------------------------------------------------------------------------------
# 5. the bars have teeth
# ------------------------------------------------------------------------------------------------------------------------------
def test_the_bars_fail_on_a_slightly_wrong_problem(variant):
    """The kernel's result on the right problem, checked with the same helpers against the oracle of a slightly wrong one (and, for
    the visibility check, with the background's gradient moved to d rgb): each must fail some bar by 10x or more, and every bar must
    fail by 10x somewhere -- so the matrix above would catch a kernel that made any of these mistakes."""
    name = "small_12x96"
    c = case(name)
    ours = run(name, True)
    right = reference(name, True)
    b = bars(name, True, right)
    ratio = lambda e: {k: e[k] / b[k] for k in b}
    assert max(ratio(errors(ours, right, c)).values()) <= 1.0
    seen = {}
    for wrong in WRONG:
        r = ratio(errors(ours, reference(name, True, wrong), c))
        print("FACTORED_TEETH " + json.dumps(dict(wrong=wrong, variant=variant, ratio={k: float("%.3g" % v) for k, v in r.items()})))
        assert max(r.values()) >= 10, (wrong, r)
        for k, v in r.items():
            seen[k] = max(seen.get(k, 0.0), v)
    moved = dict(ours, g_rgb=ours["g_rgb"] + ours["g_bg"], g_bg=np.zeros_like(ours["g_bg"]))
    r = ratio(errors(moved, right, c))
    print("FACTORED_TEETH " + json.dumps(dict(wrong="bg_gradient_sent_to_rgb", variant=variant, ratio={k: float("%.3g" % v) for k, v in r.items()})))
    assert r["g_bg_own"] >= 10 and r["g_rgb"] >= 10, r
    assert all(v >= 10 for v in seen.values()), seen
