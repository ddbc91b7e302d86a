"""The forward's two outputs besides colour and depth: the packed frames of the fused all-gather (peer_frames / n_peers /
frame_offset) and the transmittance the training forward saves for the backward (run on an H100: pytest -m gpu; the float64
reference's self-check runs without a GPU).

A. Fused-gather frames.  peer_frames is a device array of n_peers float* bases of [F,4,H,W] buffers, so local buffers run the same
   kernel code as NVLink peer buffers.  The reference is the same descriptor with color/depth outputs on the same kernel and ring
   depth, packed as [V,4,H,W]: only the store differs, so slots [off, off + V) of every buffer must equal it bit for bit, every
   other slot must keep its NaN sentinel, and the flags must be the plain call's.

B. Saved transmittance [V,N,H,W] against float64.  T64_i = prod_{j<i} (1 - a_j), with a_j the bilinear alpha (zero padding)
   computed in float64 at the texel coordinates of mpi_oracle.coords (bit-exact with the kernels').  Bound, with u = 2^-24:

       |T_i - T64_i| <= (10 i + 1) u + i 1e-10

   Per plane the kernels make these errors, each relative to a quantity <= 1 (T <= 1, the taps and the weights are in [0, 1]):
     * the bilinear weights: the direct kernel forms wx0 = RN(1 - wx1) (<= u/2) and four products (<= u each, relative), in all
       <= 2u over the four weights; the staged fast body forms w11 = RN(wx1 wy1), w10 = RN(wy1 - w11), w01 = RN(wx1 - w11),
       w00 = RN(wy0 - w01), whose errors chain, in all <= 3.5u;
     * a = the FMA chain a00 w00 + ... over the four taps: four roundings, <= 4u;  so |a - a64| <= 7.5u;
     * the update: staged T - RN(a T) (two roundings, <= 2u T), direct RN(T RN(RN(1 - a) + 1e-10)) (three, <= 1.5u T, plus the
       reference's 1e-10 T <= 1e-10).
   The error carried from plane i is multiplied by 1 - a64_i in [0, 1], so |e_{i+1}| <= |e_i| + 9.5u + 1e-10; c = 10 leaves room
   for the second-order terms and c0 = 1 for plane 0, where T is exactly 1.
   Exact properties besides: T_0 == 1; |T_{i+1}| <= |T_i|; T <= 1; rays that are NaN or have ray_z == 0 keep T == 1; the
   factored MPI's T is the expanded MPI's bit for bit (T depends on alpha only).  T is NOT always >= 0: where four alpha taps of
   1 are interpolated, the rounded weights can sum to 1 + 2^-23, as in the reference, and T steps to -2^-23 T; the bound on
   |a - a64| keeps it >= -2^-20.  T is written into a sentinel-filled allocation: every element must be written and the slack
   around it untouched.  test_transmittance_bars_fail_on_wrong_problems shows the bound fails by >= 10x on two wrong problems.

C. The training instantiations (mpi_fwd_staged_kernel<kKeyEmit | ...>, the direct kernel with transmittance set) differ from the
   inference ones only by the T stores, so their colour, depth and flags must be the inference kernel's bit for bit, through the
   descriptor and through the classic gmpi_mpi_render_fwd_train.

D. The classic entry points with data: gmpi_mpi_render_fwd is bitwise gmpi_mpi_render_fwd_ex; gmpi_mpi_render_bwd (no T: the
   two-pass direct kernel) and gmpi_mpi_render_bwd_saved (the box kernel) are within 2e-5 of the oracle's backward, also when the
   box kernel is fed the T of the direct forward (the T*((1-a)+1e-10) form)."""
import ctypes
import functools
import json

import numpy as np
import pytest
import torch

import mpi_oracle
from ml_gmpi_b200 import _lib, synth
from ml_gmpi_b200.camera import cam_params
from conftest import MPI_CASES, rel_err
from testlib import (EXPECT, GEOMETRY, assert_bitwise, case, dev, forced_kernel, kernel_fixture, on_device, oracle_backward, oracle_forward,
                     set_kernel)

gpu = pytest.mark.gpu
U = 2.0 ** -24
SENTINEL = 0x7FC0DEAD          # a quiet NaN no kernel writes
OPT_AC, OPT_CHECK, OPT_M11, OPT_ES, OPT_F16 = (_lib.OPT_ALIGN_CORNERS, _lib.OPT_CHECK_LAST_PLANE, _lib.OPT_COLOR_MINUS1_1,
                                               _lib.OPT_EARLY_STOP, _lib.OPT_MPI_F16)


# The direct kernels, or the staged forward forced at a 2- or 3-stage ring whatever the number of tiles (the factored forward keeps
# its 3-stage ring).
variant = kernel_fixture("direct", "staged2", "staged3")


def _sentinel(n):
    return torch.full((n,), SENTINEL, dtype=torch.int32, device=dev()).view(torch.float32)


def _plan(desc):
    p, why = _lib.fwd_plan(desc)
    return ("staged" if p == _lib.PLAN_STAGED else "direct"), why


def _expect_plan(variant, desc):
    """The kernel the forced variant gets: direct, or staged wherever the texture width allows it."""
    p, why = _plan(desc)
    if variant == "direct":
        assert p == "direct" and why & 16, (p, why)
    else:
        assert p == "staged" or why == 1, (p, why)     # why == 1: Wt % 4 (8 in fp16) != 0, no tensor map
    return p


# ------------------------------------------------------------------------------------------------------------------------------
# A. fused-gather frames
# ------------------------------------------------------------------------------------------------------------------------------
SHAPES = {                     # (H, W): crops of a 136^2 pinhole image
    "w128_partial_rows": (100, 128),   # (i) W % 64 == 0, partial bottom tiles
    "w136_h100": (100, 136),           # (ii) W % 4 == 0, W % 64 != 0: float4 stores with quads outside the image
    "w99_h101": (101, 99),             # (iii) W % 4 != 0: scalar peer stores
}


@functools.lru_cache(maxsize=None)
def gather_case(H, W, n_mpi=2, views=2, N=12, tex=64, img=136, seed=11):
    geo = synth.make_case(n_planes=N, tex=tex, img=img, n_mpi=n_mpi, views_per_mpi=views, seed=seed, rgba=False)
    gen = torch.Generator().manual_seed(seed)
    rgba = torch.rand((n_mpi, N, 4, tex, tex), generator=gen)
    rgba[:, :-1, 3] *= 0.3
    rgba[:, -1, 3] = 1.0
    y0, x0 = (img - H) // 2, (img - W) // 3
    ray = geo.ray_dir[:, :, y0:y0 + H, x0:x0 + W].contiguous()
    V = n_mpi * views
    cam = cam_params(geo.c2w, 1.1 * W, H, W)
    return dict(rgba=rgba, view2mpi=geo.view2mpi, dhw=geo.dhw, ray_dir=ray, eye=geo.eye, z_dir=geo.z_dir, cam=cam, V=V)


FORMS = {
    "fp32": dict(opts=OPT_AC),
    "fp32_acfalse_check_m11": dict(opts=OPT_CHECK | OPT_M11),
    "factored_bg": dict(opts=OPT_AC | OPT_M11, factored=True, bg=True),
    "factored_nobg": dict(opts=OPT_AC | OPT_CHECK, factored=True, bg=False),
    "fp16": dict(opts=OPT_AC | OPT_M11, half=True),
    "fp16_factored": dict(opts=OPT_AC, half=True, factored=True, bg=True),
    "early_stop_0": dict(opts=OPT_AC | OPT_M11, tau=0.0),
    "early_stop_2^-24": dict(opts=OPT_AC, tau=2.0 ** -24),
    "early_stop_1e-3": dict(opts=OPT_AC | OPT_CHECK | OPT_M11, tau=1e-3),
    "early_stop_1e-3_factored": dict(opts=OPT_AC, tau=1e-3, factored=True, bg=True),
    "cam": dict(opts=OPT_AC | OPT_M11, cam=True),
    "cam_factored": dict(opts=OPT_AC, cam=True, factored=True, bg=False),
    "view_group2": dict(opts=OPT_AC | OPT_M11, view_group=2),
    "view_group2_factored_cam": dict(opts=OPT_AC, view_group=2, factored=True, bg=True, cam=True),
}


def _form_inputs(c, form):
    """Descriptor fields (MPI, camera, options, sizes) of a form; tensors are kept alive in the dict."""
    f = FORMS[form]
    d = dev()
    dt = torch.float16 if f.get("half") else torch.float32
    rgba = c["rgba"].to(d)
    M, N, _, Ht, Wt = rgba.shape
    V, _, H, W = c["ray_dir"].shape
    if f.get("factored"):
        mpi = dict(rgb=rgba[:, 0, :3].contiguous().to(dt), alpha=rgba[:, :, 3:4].contiguous().to(dt),
                   bg_rgb=rgba[:, -1, :3].contiguous().to(dt) if f.get("bg") else None)
    else:
        mpi = dict(rgba=rgba.to(dt))
    cams = dict(cam=c["cam"].to(d)) if f.get("cam") else dict(ray_dir=c["ray_dir"].to(d), eye=c["eye"].to(d), z_dir=c["z_dir"].to(d))
    opts = f["opts"] | (OPT_F16 if f.get("half") else 0) | (OPT_ES if "tau" in f else 0)
    return dict(options=opts, M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, view_group=f.get("view_group", 1), early_stop=f.get("tau"),
                view2mpi=c["view2mpi"].to(d), dhw=c["dhw"].to(d), **mpi, **cams)


def _fwd(inputs, **out):
    flags = torch.zeros(1, dtype=torch.int32, device=dev())
    keep = dict(inputs, flags=flags, **out, stream=torch.cuda.current_stream().cuda_stream)
    _lib.check(_lib.load().gmpi_mpi_render_fwd_ex(ctypes.byref(_lib.make_desc(**keep))))
    torch.cuda.synchronize()
    return int(flags.item())


def packed_reference(inputs):
    """The plain call on the same kernel: (colour, depth) packed as [V,4,H,W], flags."""
    V, H, W = inputs["V"], inputs["H"], inputs["W"]
    color, depth = _sentinel(V * 3 * H * W).view(V, 3, H, W), _sentinel(V * H * W).view(V, 1, H, W)
    flags = _fwd(inputs, color=color, depth=depth)
    return torch.cat([color, depth], 1), flags


def gather(inputs, n_peers, F, offset):
    """The fused all-gather into n_peers sentinel-filled [F,4,H,W] buffers: (buffers, flags, plan of the call)."""
    H, W = inputs["H"], inputs["W"]
    bufs = [_sentinel(F * 4 * H * W).view(F, 4, H, W) for _ in range(n_peers)]
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=dev())
    out = dict(peer_frames=ptrs, n_peers=n_peers, frame_offset=offset)
    plan = _plan(_lib.make_desc(**inputs, **out))
    flags = _fwd(inputs, **out)
    return bufs, flags, plan


def check_frames(bufs, ref, offset, label):
    V = ref.shape[0]
    for r, b in enumerate(bufs):
        got = b[offset:offset + V]
        assert_bitwise(got, ref, (label, r))
        rest = torch.cat([b[:offset].flatten(), b[offset + V:].flatten()])
        assert bool((rest.view(torch.int32) == SENTINEL).all()), (label, r, "a store outside slots [offset, offset + V)")


def _gather_matrix():
    for shape in SHAPES:
        for form in FORMS:
            yield pytest.param(shape, form, id=f"{shape}-{form}")


@gpu
@pytest.mark.parametrize("shape,form", list(_gather_matrix()))
def test_fused_gather_frames_are_the_packed_plain_render(shape, form, variant):
    H, W = SHAPES[shape]
    c = gather_case(H, W)
    inputs = _form_inputs(c, form)
    p = _expect_plan(variant, _lib.make_desc(**inputs))
    if variant != "direct":
        assert p == "staged"             # Wt = 64: the staged kernel also in fp16
    ref, ref_flags = packed_reference(inputs)
    assert not bool((ref.view(torch.int32) == SENTINEL).any()), "the plain call left pixels unwritten"
    V = c["V"]
    F = V + 3
    for n_peers, offset in ((1, 0), (2, F - V), (2, 1)):
        bufs, flags, plan = gather(inputs, n_peers, F, offset)
        assert plan[0] == p, (plan, p)
        check_frames(bufs, ref, offset, (shape, form, variant, n_peers, offset))
        assert flags == ref_flags, (flags, ref_flags)


@gpu
@pytest.mark.parametrize("form", ["fp32", "factored_bg", "fp16", "early_stop_1e-3", "cam", "view_group2"])
def test_fused_gather_plans_the_staged_kernel_at_120_tiles(form):
    """4 views of 256^2 = 144 tiles of 64 x 30: the automatic choice is the staged kernel, with peer_frames set."""
    set_kernel("auto")
    c = gather_case(256, 256, n_mpi=2, views=2, N=16, tex=128, img=256, seed=12)
    inputs = _form_inputs(c, form)
    ref, ref_flags = packed_reference(inputs)
    bufs, flags, plan = gather(inputs, 2, 7, 3)
    assert plan == ("staged", 0), plan
    check_frames(bufs, ref, 3, form)
    assert flags == ref_flags


@gpu
def test_fused_gather_one_rank_of_the_two_gpu_headline():
    """One rank's share of the 2-GPU headline: 4 MPIs x 96 planes x 1024^2, frames 4..7 of two [8,4,1024,1024] buffers, automatic
    choice (the staged kernel on its 2-stage ring: every view has its own MPI, larger than L2)."""
    set_kernel("auto")
    d = dev()
    M, N, R = 4, 96, 1024
    geo = synth.make_case(n_planes=N, tex=8, img=R, n_mpi=M, seed=1234, rgba=False)
    rgba = torch.rand((M, N, 4, R, R), generator=torch.Generator(device=d).manual_seed(5), device=d)
    rgba[:, -1, 3] = 1.0
    c = dict(rgba=rgba, view2mpi=geo.view2mpi, dhw=geo.dhw, ray_dir=geo.ray_dir, eye=geo.eye, z_dir=geo.z_dir, V=M)
    inputs = dict(_form_inputs(c, "fp32"), options=OPT_AC | OPT_CHECK | OPT_M11)     # bench.py's options
    assert _lib.load().gmpi_debug_fwd_ring_stages(M, M, N, R, R, 1) == 2
    ref, ref_flags = packed_reference(inputs)
    bufs, flags, plan = gather(inputs, 2, 8, 4)
    assert plan == ("staged", 0), plan
    check_frames(bufs, ref, 4, "headline")
    assert flags == ref_flags


@gpu
def test_classic_gather_entry_point_is_bitwise_the_descriptor(variant):
    lib = _lib.load()
    c = gather_case(100, 136)
    inputs = _form_inputs(c, "fp32_acfalse_check_m11")
    ref, ref_flags = packed_reference(inputs)
    V, H, W = c["V"], 100, 136
    F, off = V + 2, 2
    bufs = [_sentinel(F * 4 * H * W).view(F, 4, H, W) for _ in range(2)]
    ptrs = torch.tensor([b.data_ptr() for b in bufs], dtype=torch.int64, device=dev())
    flags = torch.zeros(1, dtype=torch.int32, device=dev())
    i = inputs
    _lib.check(lib.gmpi_mpi_render_fwd_gather(i["rgba"].data_ptr(), i["view2mpi"].data_ptr(), i["dhw"].data_ptr(), i["ray_dir"].data_ptr(),
                                              i["eye"].data_ptr(), i["z_dir"].data_ptr(), ptrs.data_ptr(), 2, off, flags.data_ptr(),
                                              i["M"], V, i["N"], i["Ht"], i["Wt"], H, W, i["options"], None))
    torch.cuda.synchronize()
    check_frames(bufs, ref, off, ("classic", variant))
    assert int(flags.item()) == ref_flags


# ------------------------------------------------------------------------------------------------------------------------------
# B. the float64 reference of the saved transmittance
# ------------------------------------------------------------------------------------------------------------------------------
def bilinear64(tex, ix, iy):
    """F.grid_sample(bilinear, zeros) in float64: tex [V,Ht,Wt], texel coordinates ix/iy [V,H,W] -> [V,H,W].  A coordinate outside
    (-1, Wt) x (-1, Ht), or NaN, samples nothing (the kernels' coord_hits)."""
    V, Ht, Wt = tex.shape
    ix, iy = ix.astype(np.float64), iy.astype(np.float64)
    hit = (ix > -1) & (ix < Wt) & (iy > -1) & (iy < Ht)
    ix, iy = np.where(hit, ix, 0.0), np.where(hit, iy, 0.0)
    x0, y0 = np.floor(ix), np.floor(iy)
    wx1, wy1 = ix - x0, iy - y0
    flat = tex.reshape(V, -1).astype(np.float64)
    out = np.zeros(ix.shape)
    for dy, wy in ((0, 1.0 - wy1), (1, wy1)):
        for dx, wx in ((0, 1.0 - wx1), (1, wx1)):
            x, y = x0 + dx, y0 + dy
            inside = hit & (x >= 0) & (x < Wt) & (y >= 0) & (y < Ht)
            k = (np.clip(y, 0, Ht - 1) * Wt + np.clip(x, 0, Wt - 1)).astype(np.int64).reshape(V, -1)
            out += np.where(inside, wx * wy * np.take_along_axis(flat, k, axis=1).reshape(ix.shape), 0.0)
    return out


def composite64(c, alpha_scale=1.0, with_color=False):
    """T64 [V,N,H,W] (T64_i = prod_{j<i} (1 - a_j)); with_color: also the float64 colour [V,3,H,W] and depth [V,1,H,W]."""
    rgba, v2m = c["rgba"], np.asarray(c["view2mpi"], np.int64)
    M, N, _, Ht, Wt = rgba.shape
    ray = np.asarray(c["ray_dir"], np.float32)
    V, _, H, W = ray.shape
    co = mpi_oracle.coords(c["view2mpi"], c["dhw"], ray, c["eye"], Ht, Wt, align_corners=c["ac"])
    T = np.ones((V, H, W))
    Ts = np.empty((V, N, H, W))
    col, cws = np.zeros((V, 3, H, W)), np.zeros((V, H, W))
    ray64, eye64 = ray.astype(np.float64), np.asarray(c["eye"], np.float64)
    for i in range(N):
        Ts[:, i] = T
        ix, iy = co[:, i, 0], co[:, i, 1]
        a = bilinear64(rgba[v2m, i, 3], ix, iy) * alpha_scale
        if with_color:
            w = a * T
            for ch in range(3):
                col[:, ch] += w * bilinear64(rgba[v2m, i, ch], ix, iy)
            with np.errstate(divide="ignore", invalid="ignore"):
                scale = (np.asarray(c["dhw"], np.float64)[v2m, i, 0] - eye64[:, 2])[:, None, None] / ray64[:, 2]
            cws += np.where(w != 0, w * scale, 0.0)
        T = T * (1.0 - a)
    if not with_color:
        return Ts
    dz = np.einsum("vchw,vc->vhw", ray64, np.asarray(c["z_dir"], np.float64))
    return Ts, col, (cws * dz)[:, None]


def t_bound(N):
    """(10 i + 1) u + i 1e-10 of plane i (module docstring)."""
    i = np.arange(N, dtype=np.float64)
    return (10 * i + 1) * U + i * 1e-10


@pytest.mark.parametrize("name", MPI_CASES)
def test_float64_transmittance_reference_composites_the_oracle_and_golden_colours(name):
    """CPU self-check of composite64: the colour and depth it composites from its own T64 match the oracle's forward and the
    reference's golden colour and depth within 1e-6 (relative to the largest value)."""
    c = case(name)
    T64, col, dep = composite64(c, with_color=True)
    assert (T64[:, 0] == 1).all() and (T64 >= 0).all() and (T64 <= 1).all()
    oc, od, _ = oracle_forward(c, align_corners=c["ac"])
    e = dict(oracle_color=rel_err(col, oc), oracle_depth=rel_err(dep, od), golden_color=rel_err(col, c["color"]),
             golden_depth=rel_err(dep, c["depth"]))
    assert max(e.values()) <= 1e-6, e


# ------------------------------------------------------------------------------------------------------------------------------
# B / C. the training forward: saved T against float64, colour / depth / flags bitwise the inference forward
# ------------------------------------------------------------------------------------------------------------------------------
# the catalogue's cases (tests/testlib.py), and this suite's operating point: one view of a 96-plane 512^2 MPI
T_CASES = MPI_CASES + ["partial_acfalse_nonsquare", "N1", "N512", "degenerate_rays", "shuffled_rays", "corners_off_the_planes",
                       "bench_96x512_one_view"]


@functools.lru_cache(maxsize=None)
def t64(name, wrong=None):
    c = case(name)
    if wrong == "alpha_scaled":
        return composite64(c, alpha_scale=1.0 + 2.0 ** -10)
    return composite64(c)


def _train_inputs(c, factored=False):
    """Descriptor fields of a training forward of case c: its expanded MPI, or its factored MPI (whose alpha is the expanded one's)."""
    mpi = dict(zip(("rgb", "alpha", "bg_rgb"), on_device(c, "rgb", "alpha", "bg"))) if factored else dict(rgba=on_device(c, "rgba")[0])
    M, N, _, Ht, Wt = c["rgba"].shape
    V, _, H, W = c["ray_dir"].shape
    opts = (OPT_AC if c["ac"] else 0) | OPT_CHECK
    return dict(options=opts, M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, **dict(zip(GEOMETRY, on_device(c, *GEOMETRY))), **mpi)


PAD = 64                       # sentinel floats on each side of the T buffer (a multiple of 4: T stays 16-byte aligned)


def _t_buffer(V, N, H, W):
    n = V * N * H * W
    buf = _sentinel(n + 2 * PAD)
    return buf, buf[PAD:PAD + n].view(V, N, H, W)


def _check_t_buffer(buf, T, label):
    b = buf.view(torch.int32)
    assert bool((b[:PAD] == SENTINEL).all()) and bool((b[-PAD:] == SENTINEL).all()), (label, "store outside the T buffer")
    assert not bool((T.view(torch.int32) == SENTINEL).any()), (label, "T element left unwritten")


def _out(V, H, W):
    return dict(color=_sentinel(V * 3 * H * W).view(V, 3, H, W), depth=_sentinel(V * H * W).view(V, 1, H, W))


def training_forward(c, factored=False, classic=True):
    """Inference (descriptor), training (descriptor, T in a sentinel-padded buffer) and, for the expanded MPI, the classic
    gmpi_mpi_render_fwd_train and gmpi_mpi_render_fwd: colour, depth and flags must agree bit for bit.  Returns the training
    outputs (torch, on the device)."""
    inputs = _train_inputs(c, factored)
    V, N, H, W = (inputs[k] for k in ("V", "N", "H", "W"))
    inf = _out(V, H, W)
    inf_flags = _fwd(inputs, **inf)
    tr = _out(V, H, W)
    buf, T = _t_buffer(V, N, H, W)
    tr_flags = _fwd(inputs, transmittance=T, **tr)
    _check_t_buffer(buf, T, "descriptor")
    for k in ("color", "depth"):
        assert_bitwise(tr[k], inf[k], (k, "training forward != inference forward"))
    assert tr_flags == inf_flags
    if classic and not factored:
        lib = _lib.load()
        i = inputs
        geo = [i[k].data_ptr() for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")]
        sizes = [i["M"], V, N, i["Ht"], i["Wt"], H, W, i["options"]]
        ct = _out(V, H, W)
        cbuf, cT = _t_buffer(V, N, H, W)
        cflags = torch.zeros(1, dtype=torch.int32, device=dev())
        _lib.check(lib.gmpi_mpi_render_fwd_train(*geo, ct["color"].data_ptr(), ct["depth"].data_ptr(), cT.data_ptr(), cflags.data_ptr(),
                                                 *sizes, None))
        cf = _out(V, H, W)
        fflags = torch.zeros(1, dtype=torch.int32, device=dev())
        _lib.check(lib.gmpi_mpi_render_fwd(*geo, cf["color"].data_ptr(), cf["depth"].data_ptr(), fflags.data_ptr(), *sizes, None))
        torch.cuda.synchronize()
        _check_t_buffer(cbuf, cT, "gmpi_mpi_render_fwd_train")
        assert_bitwise(cT, T, "gmpi_mpi_render_fwd_train T != descriptor T")
        for k in ("color", "depth"):
            assert_bitwise(ct[k], inf[k], (k, "gmpi_mpi_render_fwd_train != inference forward"))
            assert_bitwise(cf[k], inf[k], (k, "gmpi_mpi_render_fwd != gmpi_mpi_render_fwd_ex"))
        assert int(cflags.item()) == inf_flags and int(fflags.item()) == inf_flags
    return dict(T=T, flags=tr_flags, plan=_plan(_lib.make_desc(**inputs))[0], **tr)


def t_errors(T, ref):
    """max over elements of |T - T64| / bound, and the largest |T - T64|."""
    err = np.abs(T.astype(np.float64) - ref)
    return float((err / t_bound(ref.shape[1])[None, :, None, None]).max()), float(err.max())


def check_t_properties(T, label):
    assert (T[:, 0] == 1).all(), label
    assert T.max() <= 1 and T.min() >= -2.0 ** -20, (label, float(T.min()), float(T.max()))
    assert (np.abs(T[:, 1:]) <= np.abs(T[:, :-1])).all(), (label, "|T| increased from one plane to the next")


@gpu
@pytest.mark.parametrize("name", T_CASES)
def test_saved_transmittance_against_float64_and_training_equals_inference(name, variant):
    c = case(name)
    ours = training_forward(c)
    if variant != "direct":
        assert ours["plan"] == "staged" or c["rgba"].shape[-1] % 4, ours["plan"]
    T = ours["T"].cpu().numpy()
    ref = t64(name)
    ratio, worst = t_errors(T, ref)
    print("TRANSMITTANCE " + json.dumps(dict(case=name, variant=variant, plan=ours["plan"], err_over_bar=float("%.3g" % ratio),
                                             max_abs_err=float("%.3g" % worst), min_T=float(T.min()))))
    check_t_properties(T, (name, variant))
    assert ratio <= 1.0, (name, variant, ratio, worst)
    if "ok" in c:                  # rays that are NaN or parallel to the planes
        assert (T.transpose(1, 0, 2, 3)[:, ~c["ok"]] == 1).all(), T.transpose(1, 0, 2, 3)[:, ~c["ok"]]
    fac = training_forward(c, factored=True)
    assert fac["plan"] == ours["plan"] or variant == "direct"
    assert_bitwise(fac["T"], ours["T"], (name, variant, "factored T != expanded T"))


@gpu
def test_transmittance_bars_fail_on_wrong_problems(variant):
    """The bound of the right problem holds; against T shifted by one plane and against alpha scaled by 1 + 2^-10 it fails by 10x
    or more."""
    name = "small_12x96"
    T = training_forward(case(name), classic=False)["T"].cpu().numpy()
    right = t64(name)
    assert t_errors(T, right)[0] <= 1.0
    shifted = np.concatenate([right[:, 1:], right[:, -1:]], 1)
    ratios = dict(shifted_one_plane=t_errors(T, shifted)[0], alpha_scaled=t_errors(T, t64(name, "alpha_scaled"))[0])
    print("TRANSMITTANCE_TEETH " + json.dumps(dict(variant=variant, ratio={k: float("%.3g" % v) for k, v in ratios.items()})))
    assert all(r >= 10 for r in ratios.values()), ratios


# ------------------------------------------------------------------------------------------------------------------------------
# D. the classic backward entry points with data
# ------------------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["tiny_2mpi_3view", "staged_shape"])
def test_classic_backward_entry_points_match_the_oracle(name):
    """gmpi_mpi_render_bwd (two-pass direct kernel), gmpi_mpi_render_bwd_saved with the direct forward's T (direct kernels forced,
    and the box kernel) and with the staged forward's T (box kernel): each within EXPECT of the oracle's backward."""
    c = case(name)
    lib = _lib.load()
    V, _, H, W = c["ray_dir"].shape
    ref = oracle_backward(c, c["gc"], c["gd"], align_corners=c["ac"])
    i = _train_inputs(c)
    geo = [i[k].data_ptr() for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")]
    sizes = [i["M"], V, i["N"], i["Ht"], i["Wt"], H, W]
    g_color, g_depth = on_device(c, "gc", "gd")
    st = torch.cuda.current_stream().cuda_stream

    def train_t():
        T = torch.empty((V, i["N"], H, W), device=dev())
        o = _out(V, H, W)
        fl = torch.zeros(1, dtype=torch.int32, device=dev())
        _lib.check(lib.gmpi_mpi_render_fwd_train(*geo, o["color"].data_ptr(), o["depth"].data_ptr(), T.data_ptr(), fl.data_ptr(), *sizes,
                                                 i["options"], st))
        return T

    def bwd(T=None):
        g = torch.full_like(i["rgba"], float("nan"))
        opt = i["options"] | _lib.OPT_ZERO_GRAD
        if T is None:
            _lib.check(lib.gmpi_mpi_render_bwd(*geo, g_color.data_ptr(), g_depth.data_ptr(), g.data_ptr(), *sizes, opt, st))
        else:
            _lib.check(lib.gmpi_mpi_render_bwd_saved(*geo, T.data_ptr(), g_color.data_ptr(), g_depth.data_ptr(), g.data_ptr(), *sizes,
                                                     opt, st))
        torch.cuda.synchronize()
        return g.cpu().numpy()

    with forced_kernel("direct"):
        T_direct = train_t()
        grads = dict(bwd_two_pass=bwd(), bwd_saved_direct=bwd(T_direct))
    with forced_kernel("staged3"):
        assert _plan(_lib.make_desc(**i))[0] == "staged"
        T_staged = train_t()
        grads.update(bwd_saved_box=bwd(T_staged), bwd_saved_box_direct_T=bwd(T_direct))
    e = {k: rel_err(v, ref) for k, v in grads.items()}
    print("CLASSIC_BWD " + json.dumps(dict(case=name, err={k: float("%.3g" % v) for k, v in e.items()},
                                           T_forms_differ=float((T_direct - T_staged).abs().max()))))
    assert all(np.isfinite(v).all() for v in grads.values())
    assert max(e.values()) <= EXPECT, e
