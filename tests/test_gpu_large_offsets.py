"""A render or a gradient must not depend on where its MPI, view or output slab sits in its buffer, also past 2^31 elements.

The C ABI takes M*N < 2^31 planes of Ht*Wt < 2^31 texels, so every element offset is 64-bit.  Each test runs one call shape twice:
near (the content at the start of its buffer: MPI slot 0, view 0, frame 0) and far (at the end, past 2^31 elements), with every
other MPI slot NaN (a read from a wrong address shows up in the output) and the gradients zeroed by the call (GMPI_ZERO_GRAD: a
stray write shows up in a slab no view touches).  The forward and the deterministic backward are bitwise the same near and far; the
default backward differs only in the order of its fp32 atomics.  The far result is then anchored to the oracle on the one MPI and
its views.  tests/test_large_offsets.py checks, on the CPU, that these shapes put the planes the fast and the generic bodies read
past 2^31 and that each test's peak fits 24 GiB.

Each test skips unless the card has its declared peak free, prints "LARGE_OFFSETS {...}" (its measured peak, wall time and card),
and fails if it held more than it declared."""
import ctypes
import json
import time

import numpy as np
import pytest
import torch

import mpi_oracle
import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth
from ml_gmpi_b200.camera import cam_params, focal_from_fov, sphere_poses
from ml_gmpi_b200.geometry import FFHQ
from conftest import rel_err
from testlib import (BIG_IMG, BIG_M, BIG_M_FACTORED, BIG_N, BIG_PEAK_BYTES, BIG_R, BIG_SLACK, BIG_V_COLOR, BIG_V_GATHER, EXPECT,
                     SMALL_MPI, assert_bitwise, big_views, dev, factored_refs, forced_kernel, headline_case, kernel_fixture,
                     native_vs_fp32, oracle_backward, oracle_forward, render_fwd, set_kernel, skip_stats, upstream)

pytestmark = pytest.mark.gpu
NEAR_FAR = 1e-6     # near against far where only the order of fp32 atomics differs
N, R, M, MF = BIG_N, BIG_R, BIG_M, BIG_M_FACTORED
variant = kernel_fixture("auto", "direct")


@pytest.fixture
def budget(request):
    """budget(key) skips the test unless the card has BIG_PEAK_BYTES[key] free; afterwards the test must not have held more."""
    keys = []

    def room(key):
        need = BIG_PEAK_BYTES[key] + BIG_SLACK
        free = torch.cuda.mem_get_info()[0]
        if free < need:
            pytest.skip(f"needs {need / 1e9:.1f} GB, {free / 1e9:.1f} GB free")
        keys.append(key)

    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    base, t0 = torch.cuda.memory_allocated(), time.perf_counter()
    yield room
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    torch.cuda.empty_cache()
    print("LARGE_OFFSETS " + json.dumps(dict(test=request.node.name, peak_gb=round(peak / 1e9, 2),
                                             declared_gb=round(BIG_PEAK_BYTES[keys[0]] / 1e9, 2) if keys else None,
                                             seconds=round(time.perf_counter() - t0, 1), gpu=torch.cuda.get_device_name())))
    if keys:
        assert peak <= BIG_PEAK_BYTES[keys[0]] + BIG_SLACK, (keys[0], peak)


def _views(slot, n_mpi, views=(0, 1)):
    """big_views' views `views`, of MPI `slot` of an n_mpi-MPI buffer."""
    v = big_views()
    sel = list(views)
    return dict(v, view2mpi=np.full(len(sel), slot, np.int32), dhw=np.repeat(v["dhw"], n_mpi, 0), ray_dir=v["ray_dir"][sel],
                eye=v["eye"][sel], z_dir=v["z_dir"][sel])


def _content():
    """The headline MPI (testlib.headline_case: 96 x 1024^2, equal-weight alpha) on the device, [N,4,R,R] fp32."""
    return torch.from_numpy(headline_case()["rgba"][0]).to(dev())


def _native(x32, dtype):
    """(the MPI as `dtype` renders it natively, its fp32 conversion): fp16, or uint8 codes round(255 x)."""
    if dtype == "fp32":
        return x32, x32
    if dtype == "fp16":
        h = x32.half()
        return h, h.float()
    u = (x32 * 255).round_().to(torch.uint8)
    return u, _unorm8_conversion(u)


def _unorm8_conversion(u):
    """g.unorm8_to_float(u), plane by plane: its table lookup holds int32 and int64 indices of every code at once."""
    out = torch.empty(u.shape, device=u.device)
    for p_out, p_in in zip(out.view(-1, R, R), u.view(-1, R, R)):
        p_out.copy_(g.unorm8_to_float(p_in))
    return out


_FILL = {"fp32": float("nan"), "fp16": float("nan"), "uint8": 255}    # uint8 has no NaN: the other slots are opaque white
_DTYPE = {"fp32": torch.float32, "fp16": torch.float16, "uint8": torch.uint8}


def _move(buf, src, dst, fill):
    """MPI slot src of buf to slot dst; slot src gets the fill."""
    buf[dst].copy_(buf[src])
    buf[src].fill_(fill)


def _ring_kernel(M_, V):
    """The kernel name (testlib.KERNELS) that renders like the automatic choice for M_ MPIs and V views of the big MPI."""
    return "staged%d" % _lib.load().gmpi_debug_fwd_ring_stages(M_, V, N, R, R, 1)


def _minus1_1(c):
    return 2.0 * c.astype(np.float64) - 1.0


_oracle_cache = {}


@pytest.fixture(scope="module", autouse=True)
def _drop_oracle_cache():
    """The oracle's results are shared by this module's tests only: its backward is a 1.6 GB gradient."""
    yield
    _oracle_cache.clear()


def _oracle_forward():
    """(colour in [-1, 1], depth) of the oracle on the headline MPI alone, both views of big_views."""
    if "fwd" not in _oracle_cache:
        rc, rd, _ = oracle_forward(big_views(), rgba=headline_case()["rgba"])
        _oracle_cache["fwd"] = (_minus1_1(rc), rd)
    return _oracle_cache["fwd"]


def _oracle_backward(views):
    """d rgba of the oracle on the headline MPI alone, big_views' views `views`, under upstream(len(views), R, R, 3)'s gradients
    (colour in [0, 1])."""
    if ("bwd", views) not in _oracle_cache:
        gc, gd = upstream(len(views), R, R, 3)
        _oracle_cache["bwd", views] = oracle_backward(_views(0, 1, views), gc, gd, rgba=headline_case()["rgba"])[0]
    return _oracle_cache["bwd", views]


def _max_abs(a, b):
    """(max |a - b|, max |b|) of two tensors or arrays of the same shape, slice by slice on the device in float64 (a 1.6 GB MPI is
    3.2 GB in float64); NaN anywhere in a makes the first inf."""
    d = dev()
    t = lambda x, i: (torch.from_numpy(np.ascontiguousarray(x[i])) if isinstance(x, np.ndarray) else x[i]).to(d, torch.float64)
    num = den = 0.0
    for i in range(a.shape[0]):
        x, y = t(a, i), t(b, i)
        if torch.isnan(x).any():
            return float("inf"), float("nan")
        num, den = max(num, float((x - y).abs().max())), max(den, float(y.abs().max()))
    return num, den


def _rel(a, b):
    """rel_err (conftest) of two tensors or arrays, computed by _max_abs; NaN anywhere in a makes it inf."""
    num, den = _max_abs(a, b)
    return num if num == float("inf") else num / (den if den > 0 else 1.0)


def _most_taps(v):
    """(front, last): the largest number of bilinear taps a texel of the planes in front of the last, and of the last plane,
    receives from the views v (the oracle's texel coordinates).  The factored colour gradients sum that many fixed-point roundings
    (tests/test_gpu_factored.py, bars)."""
    c = mpi_oracle.coords(v["view2mpi"], v["dhw"], v["ray_dir"], v["eye"], R, R, v["ac"])
    front, last = np.zeros(R * R, np.int64), np.zeros(R * R, np.int64)
    for i in range(N):
        ix, iy = c[:, i, 0].ravel(), c[:, i, 1].ravel()
        ok = np.isfinite(ix) & np.isfinite(iy)
        x0, y0 = (np.floor(np.clip(a[ok], -2, R + 1)).astype(np.int64) for a in (ix, iy))
        hist = front if i < N - 1 else last
        for dy in (0, 1):
            for dx in (0, 1):
                x, y = x0 + dx, y0 + dy
                inside = (x >= 0) & (x < R) & (y >= 0) & (y < R)
                hist += np.bincount((y * R + x)[inside], minlength=R * R)
    return int(front.max()), int(last.max())


def _all_plus_zero(x):
    """Every element of the fp32 tensor x is +0 (bit pattern 0)."""
    return not bool(x.view(torch.int32).any())


# ------------------------------------------------------------------------------------------------------------------------------
# forward: expanded fp32 / fp16 / uint8 MPIs, early stop, empty-space skipping
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("dtype", ["fp32", "fp16", "uint8"])
def test_expanded_forward_near_equals_far(dtype, variant, budget):
    """M = 6 MPIs of 96 x 1024^2 (9.7 / 4.8 / 2.4 GB): MPI 0 against MPI 5, whose planes 32..95 lie past 2^31, seen from the pinhole
    view (the staged forward's fast bodies) and from shuffled rays (its generic bodies), with and without early stop (tau = 1e-3).
    Far against the oracle (fp32) or against the render of the fp32 conversion in a fresh allocation (fp16, uint8)."""
    budget(f"expanded_forward-{dtype}")
    x32 = _content()
    native, conv = _native(x32, dtype)
    big = torch.full((M, N, 4, R, R), _FILL[dtype], dtype=_DTYPE[dtype], device=dev())
    big[0].copy_(native)
    if dtype != "fp32":
        del x32
        native = None
    near = render_fwd(_views(0, M), {"rgba": big}), render_fwd(_views(0, M), {"rgba": big}, tau=1e-3)
    _move(big, 0, M - 1, _FILL[dtype])
    far = render_fwd(_views(M - 1, M), {"rgba": big}), render_fwd(_views(M - 1, M), {"rgba": big}, tau=1e-3)
    assert_bitwise(near, far, "near != far")
    del big
    torch.cuda.empty_cache()
    if dtype == "fp32":
        rc, rd = _oracle_forward()
        for v in range(2):
            assert rel_err(far[0][0][v], rc[v]) <= EXPECT and rel_err(far[0][1][v], rd[v]) <= EXPECT, v
    else:
        assert _ring_kernel(M, 2) == "staged2"       # two views of an MPI larger than L2, which alone would get the 3-stage ring
        with forced_kernel("direct" if variant == "direct" else _ring_kernel(M, 2)):
            one = render_fwd(_views(0, 1), {"rgba": conv[None]})
        assert_bitwise(far[0], one, "native != its fp32 conversion")


def test_the_comparisons_fail_on_what_a_wrapped_offset_would_read(budget):
    """What a 32-bit offset would have read instead of plane 40 of the far MPI: the NaN fill of another slot, or another MPI's
    plane.  Rendered as the near placement of that slightly wrong input, each must differ from the far render and fail the oracle's
    bar by 10x or more, so the near-against-far and oracle comparisons above would catch such a read."""
    budget("wrong_inputs")
    set_kernel("auto")
    big = torch.full((M, N, 4, R, R), float("nan"), device=dev())
    big[M - 1].copy_(_content())
    far = render_fwd(_views(M - 1, M), {"rgba": big})
    rc, _ = _oracle_forward()
    assert rel_err(far[0], rc) <= EXPECT
    other = synth.make_case(n_planes=N, tex=R, img=8, n_mpi=1, seed=99, alpha="equal_weight", device=dev()).rgba[0, 40]
    ratios = {}
    for name, plane in (("nan_fill", torch.full_like(other, float("nan"))), ("another_mpi", other)):
        big[0].copy_(big[M - 1])
        big[0, 40].copy_(plane)
        wrong = render_fwd(_views(0, M), {"rgba": big})
        with pytest.raises(AssertionError):
            assert_bitwise(wrong, far)
        ratios[name] = min(_rel(wrong[0][v:v + 1], rc[v:v + 1]) for v in range(2)) / EXPECT
    print("LARGE_OFFSETS_TEETH " + json.dumps({k: float("%.3g" % v) for k, v in ratios.items()}))
    assert all(v >= 10 for v in ratios.values()), ratios


def test_skipping_near_equals_far(budget):
    """The occupancy map of the whole M = 6 stack (NaN counts as occupied): the far MPI's words are the near MPI's, and the skipping
    render is bitwise the plain one, near and far.  The MPI is the headline one with the left quarter of every plane but the last
    transparent, so that stages are skipped."""
    budget("skipping")
    big = torch.full((M, N, 4, R, R), float("nan"), device=dev())
    big[0].copy_(_content())
    big[0, :-1, 3, :, :R // 4] = 0.0
    v = {k: torch.from_numpy(a).to(dev()) if isinstance(a, np.ndarray) else a for k, a in _views(0, M).items()}
    out = {}
    for slot in (0, M - 1):
        v2m = torch.full((2,), slot, dtype=torch.int32, device=dev())
        occ = g.build_occupancy(rgba=big)
        words = occ.occ.view(M, -1)[slot].clone()
        plain = g.render_views(big, v["dhw"], v2m, v["ray_dir"], v["eye"], v["z_dir"])
        skip = g.render_views(big, v["dhw"], v2m, v["ray_dir"], v["eye"], v["z_dir"], skip_empty=occ)
        assert skip_stats()[0] > 0
        assert_bitwise(skip, plain, ("skip != plain", slot))
        out[slot] = (words, plain)
        del occ
        if slot == 0:
            _move(big, 0, M - 1, float("nan"))
    assert_bitwise(out[0], out[M - 1], "near != far")


# ------------------------------------------------------------------------------------------------------------------------------
# backward: expanded, factored, saved transmittance
# ------------------------------------------------------------------------------------------------------------------------------
def test_expanded_backward_near_equals_far(variant, budget):
    """g_rgba of M = 6 MPIs (9.7 GB, and 9.7 GB of rgba): the two views of MPI 0 against those of MPI 5, through the default box
    backward (auto) or the direct one.  The pinhole view's stages take the box backward's fast body, the shuffled view's its generic
    body, so both bodies scatter into planes 32..95 of MPI 5, past 2^31.  Every slab of another MPI stays +0."""
    budget("expanded_backward")
    big = torch.full((M, N, 4, R, R), float("nan"), device=dev())
    big[0].copy_(_content())
    big.requires_grad_(True)
    gc, gd = upstream(2, R, R, 3, device=dev())
    kept = {}
    for slot in (0, M - 1):
        v = {k: torch.from_numpy(a).to(dev()) for k, a in _views(slot, M).items() if isinstance(a, np.ndarray)}
        color, depth = g.render_views(big, v["dhw"], v["view2mpi"], v["ray_dir"], v["eye"], v["z_dir"])
        ((color * gc).sum() + (depth * gd).sum()).backward()
        grad = big.grad
        big.grad = None
        del color, depth
        for m in range(M):
            if m != slot:
                assert _all_plus_zero(grad[m]), (slot, m)
        kept[slot] = grad[slot].cpu()
        del grad
        if slot == 0:
            with torch.no_grad():
                _move(big, 0, M - 1, float("nan"))
    del big
    assert _rel(kept[M - 1], kept[0]) <= NEAR_FAR
    assert _rel(kept[M - 1], _oracle_backward((0, 1))) <= EXPECT


def _factored(d):
    gen = torch.Generator(device=d).manual_seed(11)
    rgb, bg = torch.rand((1, 3, R, R), generator=gen, device=d), torch.rand((1, 3, R, R), generator=gen, device=d)
    return rgb, synth.equal_weight_alpha((1, N, R, R), gen, d).unsqueeze(2), bg


def test_factored_near_equals_far(budget):
    """Factored alpha and g_alpha [22, 96, 1, 1024^2] fp32 (8.9 GB each; planes 32..95 of MPI 21 lie past 2^31), with bg_rgb: the
    fp16 and the fp32 forward near = far bitwise; the fp32 backward's g_rgb, g_alpha and g_bg_rgb near and far within 1e-6 and
    against the oracle of the expanded form."""
    budget("factored")
    d = dev()
    one = _factored(d)
    shapes = ((MF, 3, R, R), (MF, N, 1, R, R), (MF, 3, R, R))
    for dt in (torch.float16, torch.float32):
        mpi = [torch.full(s, float("nan"), dtype=dt, device=d) for s in shapes]
        for t, x in zip(mpi, one):
            t[0].copy_(x[0])
        fields = lambda: dict(rgb=mpi[0], alpha=mpi[1], bg_rgb=mpi[2])
        near = render_fwd(_views(0, MF), fields())
        for t in mpi:
            _move(t, 0, MF - 1, float("nan"))
        assert_bitwise(near, render_fwd(_views(MF - 1, MF), fields()), (dt, "near != far"))
        del near
        if dt == torch.float16:
            del mpi
    gc, gd = upstream(2, R, R, 3, device=d)
    kept = {}
    for slot in (MF - 1, 0):
        leaves = [t.requires_grad_(True) for t in mpi]
        v = {k: torch.from_numpy(a).to(d) for k, a in _views(slot, MF).items() if isinstance(a, np.ndarray)}
        color, depth = g.render_views_factored(leaves[0], leaves[1], v["dhw"], v["view2mpi"], v["ray_dir"], v["eye"], v["z_dir"],
                                               bg_rgb=leaves[2])
        ((color * gc).sum() + (depth * gd).sum()).backward()
        del color, depth
        grads = [t.grad for t in leaves]
        for t in leaves:
            t.grad = None
        for m in range(MF):
            if m != slot:
                assert all(_all_plus_zero(x[m]) for x in grads), (slot, m)
        kept[slot] = [x[slot:slot + 1].cpu() for x in grads]
        del grads
        if slot == MF - 1:
            with torch.no_grad():
                for t in mpi:
                    _move(t, MF - 1, 0, float("nan"))
    del mpi, leaves
    h, v = [x.cpu() for x in one], _views(0, 1)
    ref = oracle_backward(v, gc, gd, rgba=g.expand_factored(*h))
    refs = factored_refs(ref)
    # the bars of tests/test_gpu_factored.py: relative to the largest expanded gradient S, the colour gradients add the rounding of
    # each tap's fixed-point contribution (2^-21 of the largest upstream colour gradient) to the parity bar
    kf, kl = _most_taps(v)
    S, gmax = float(np.abs(ref).max()), float(gc.abs().max())
    tols = [kf * 2.0 ** -21 * gmax / S + EXPECT, EXPECT, kl * 2.0 ** -21 * gmax / S + EXPECT]
    for k, (far, near, r, tol) in enumerate(zip(kept[MF - 1], kept[0], refs, tols)):
        assert _rel(far, near) <= NEAR_FAR, k
        err = _rel(far, r) if k == 1 else _max_abs(far, r)[0] / S
        assert err <= tol, (k, err, tol)


@pytest.mark.parametrize("twin", [0, 1], ids=["pinhole", "shuffled"])
def test_saved_transmittance_past_2_31(twin, budget):
    """The training forward of 22 views of one MPI saves T [22, 96, 1024^2] (8.9 GB; planes 32..95 of view 21 lie past 2^31).  Views
    0 and 21 are the same view of big_views (the pinhole one, whose stages take the fast bodies, or the shuffled one, whose stages take
    the generic bodies): view 21's T slab and colour are view 0's, bitwise; the backward from an upstream gradient on view 0 only,
    then on view 21 only, is bitwise the same in the deterministic backward (3.2 GB of sums) and within 1e-6 in the default box
    backward, which is within the parity bar of the oracle."""
    budget("saved_transmittance")
    d = dev()
    V = MF
    others = synth.make_case(n_planes=N, tex=8, img=R, n_mpi=1, views_per_mpi=V - 2, seed=17, rgba=False)
    v = _views(0, 1, (twin,))
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(d)
    ray = t(np.concatenate([v["ray_dir"], others.ray_dir.numpy(), v["ray_dir"]]))
    eye = t(np.concatenate([v["eye"], others.eye.numpy(), v["eye"]]))
    z = t(np.concatenate([v["z_dir"], others.z_dir.numpy(), v["z_dir"]]))
    rgba = _content()[None]
    trans = torch.full((V, N, R, R), float("nan"), device=d)
    color, depth = torch.empty((V, 3, R, R), device=d), torch.empty((V, 1, R, R), device=d)
    common = dict(M=1, V=V, N=N, Ht=R, Wt=R, H=R, W=R, rgba=rgba, view2mpi=torch.zeros(V, dtype=torch.int32, device=d), dhw=t(v["dhw"]),
                  ray_dir=ray, eye=eye, z_dir=z, transmittance=trans, flags=torch.zeros(1, dtype=torch.int32, device=d))
    lib = _lib.load()
    _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(_lib.make_desc(options=_lib.OPT_ALIGN_CORNERS, color=color, depth=depth,
                                                                       **common))))
    torch.cuda.synchronize()
    assert torch.equal(trans[V - 1].view(torch.int32), trans[0].view(torch.int32))
    assert_bitwise((color[V - 1], depth[V - 1]), (color[0], depth[0]), "view 21 != view 0")
    del color, depth
    gc1, gd1 = upstream(1, R, R, 3)
    g_rgba = torch.full_like(rgba, float("nan"))
    grads = {}
    for det in (True, False):
        for view in (0, V - 1):
            gc, gd = torch.zeros((V, 3, R, R), device=d), torch.zeros((V, 1, R, R), device=d)
            gc[view], gd[view] = gc1[0].to(d), gd1[0].to(d)
            desc = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_ZERO_GRAD, g_color=gc, g_depth=gd, g_rgba=g_rgba, **common)
            if det:
                nbytes = _lib.deterministic_scratch_bytes(desc)
                scratch = torch.empty(nbytes, dtype=torch.uint8, device=d)
                _lib.check(lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(desc), scratch.data_ptr(), nbytes))
                torch.cuda.synchronize()
                del scratch
            else:
                _lib.check(lib.gmpi_mpi_render_bwd_ex(ctypes.byref(desc)))
            del gc, gd
            grads[det, view] = g_rgba[0].cpu()
    assert_bitwise(grads[True, 0], grads[True, V - 1], "deterministic: view 21 != view 0")
    assert _rel(grads[False, V - 1], grads[False, 0]) <= NEAR_FAR
    assert _rel(grads[False, V - 1], _oracle_backward((twin,))) <= EXPECT
    assert _rel(grads[True, V - 1], _oracle_backward((twin,))) <= EXPECT


# ------------------------------------------------------------------------------------------------------------------------------
# outputs past 2^31 elements: colour and depth, uint8 video frames, fused-gather frames
# ------------------------------------------------------------------------------------------------------------------------------
_SENTINEL = {"color": -7.0, "video": 0xA5, "gather": -7.0}


def _padded(n, dtype, fill):
    """(a buffer of `fill`, its n elements in the middle) with 4096 sentinels after the n and, in front of them, 4096 or -- when n
    passes 2^31 -- 2^31: where a store whose offset wrapped as a signed 32-bit number lands."""
    lead = 1 << 31 if n > 1 << 31 else 4096
    buf = torch.full((lead + n + 4096,), fill, dtype=dtype, device=dev())
    return buf, buf[lead:lead + n]


def _all_equal(x, value):
    """Every element of the flat tensor x is `value`, tested 2^26 elements at a time (the comparison's bool tensor stays small)."""
    return all(bool((x[i:i + (1 << 26)] == value).all()) for i in range(0, x.numel(), 1 << 26))


@pytest.mark.parametrize("kind", ["color", "video", "gather"])
def test_outputs_past_2_31(kind, variant, budget):
    """Colour [684, 3, 1024^2] (8.6 GB; view 683 starts past 2^31), uint8 video frames [684, 1024^2, 3] (view 683 past 2^31 bytes)
    and fused-gather frames [513, 4, 1024^2] (frame 512 starts at 2^31), rendered from in-kernel camera rays (no ray tensor) of a
    small MPI.  Views 0 and V - 1 are twins: their frames are bitwise equal, the frames past 2^31 hold no sentinel, and the sentinels
    around the frames are untouched (_padded)."""
    budget(f"outputs-{kind}")
    d = dev()
    V = BIG_V_GATHER if kind == "gather" else BIG_V_COLOR
    yaws = torch.linspace(-0.5, 0.5, V)
    yaws[-1] = yaws[0]
    cam = cam_params(sphere_poses(yaws, torch.zeros(V), FFHQ["sphere_center"], FFHQ["sphere_r"]), focal_from_fov(FFHQ["fov_deg"], R),
                     R, R).to(d)
    small = synth.make_case(n_planes=SMALL_MPI["N"], tex=SMALL_MPI["R"], img=8, n_mpi=1, seed=23, last_alpha_one=True, device=d)
    opts = _lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1
    common = dict(M=1, V=V, N=SMALL_MPI["N"], Ht=SMALL_MPI["R"], Wt=SMALL_MPI["R"], H=R, W=R, rgba=small.rgba, dhw=small.dhw,
                  view2mpi=torch.zeros(V, dtype=torch.int32, device=d), cam=cam, flags=torch.zeros(1, dtype=torch.int32, device=d))
    s = _SENTINEL[kind]
    if kind == "color":
        bufs = [_padded(V * 3 * BIG_IMG, torch.float32, s), _padded(V * BIG_IMG, torch.float32, s)]
        frames = [bufs[0][1].view(V, 3, R, R), bufs[1][1].view(V, 1, R, R)]
        desc = _lib.make_desc(options=opts, color=frames[0], depth=frames[1], **common)
    elif kind == "video":
        bufs = [_padded(V * BIG_IMG * 3, torch.uint8, s), _padded(V * BIG_IMG, torch.uint8, s)]
        frames = [bufs[0][1].view(V, R, R, 3), bufs[1][1].view(V, R, R, 1)]
        desc = _lib.make_desc(options=opts, video_rgb=frames[0], video_depth=frames[1], depth_near=0.9,
                              depth_range=float(np.float32(0.3)), **common)
    else:
        bufs = [_padded(V * 4 * BIG_IMG, torch.float32, s)]
        frames = [bufs[0][1].view(V, 4, R, R)]
        ptrs = torch.tensor([frames[0].data_ptr()], dtype=torch.int64, device=d)
        desc = _lib.make_desc(options=opts, peer_frames=ptrs, n_peers=1, frame_offset=0, **common)
    _lib.check(_lib.load().gmpi_mpi_render_fwd_ex(ctypes.byref(desc)))
    torch.cuda.synchronize()
    for (buf, f0), f in zip(bufs, frames):
        assert torch.equal(f[V - 1], f[0]), kind
        lead = (f0.data_ptr() - buf.data_ptr()) // f0.element_size()
        assert _all_equal(buf[:lead], s) and _all_equal(buf[lead + f.numel():], s), kind
        if f.numel() > 1 << 31 and kind != "video":      # every uint8 code is a possible output
            first_far = (1 << 31) // f[0].numel()        # the first frame that reaches past 2^31 elements
            assert not bool((f[first_far:] == s).any()), kind
    assert frames[0].numel() > 1 << 31


# ------------------------------------------------------------------------------------------------------------------------------
# the range check and the occupancy build's fused flags
# ------------------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("path", ["vector", "scalar"])
@pytest.mark.parametrize("dtype", ["fp32", "fp16"])
def test_range_flags_past_2_31(dtype, path, budget):
    """M = 6 MPIs of 96 planes in [0, 1], 1024^2 (16-byte loads) or 1023^2 (a slab that is not a whole number of them: the scalar
    loop), with one value out of range at element 2^31 (a colour channel), then one more at the last element (alpha): the exact
    flag words of gmpi_mpi_check_range(_f16) and of the occupancy build."""
    budget(f"range_check-{dtype}-{path}")
    d = dev()
    side = R if path == "vector" else R - 1
    big = torch.full((M, N, 4, side, side), 0.5, dtype=_DTYPE[dtype], device=d)
    flat = big.view(-1)
    check = _lib.load().gmpi_mpi_check_range if dtype == "fp32" else _lib.load().gmpi_mpi_check_range_f16

    def flag_words():
        f1, f2 = torch.zeros(1, dtype=torch.int32, device=d), torch.zeros(1, dtype=torch.int32, device=d)
        _lib.check(check(big.data_ptr(), M, N, side, side, f1.data_ptr(), None))
        occ = g.build_occupancy(rgba=big, flags=f2)
        del occ
        return int(f1.item()), int(f2.item())

    assert flag_words() == (0, 0)
    flat[1 << 31] = 1.5
    assert flag_words() == (_lib.FLAG_RGBA_RANGE,) * 2
    flat[-1] = -0.5
    assert flag_words() == (_lib.FLAG_RGBA_RANGE | _lib.FLAG_ALPHA_RANGE,) * 2


# ------------------------------------------------------------------------------------------------------------------------------
# the host entry point
# ------------------------------------------------------------------------------------------------------------------------------
def test_host_entry_point_far_mpi(budget):
    """gmpi_mpi_render_host_ex of a uint8 host buffer of M = 6 MPIs (2.4 GB of host memory), one view of MPI 5 (its bytes start at
    2,013,265,920 and end past 2^31): bitwise the device render of that MPI alone."""
    budget("host_entry_point")
    set_kernel("auto")
    host = np.full((M, N, 4, R, R), 255, np.uint8)
    host[M - 1] = np.rint(headline_case()["rgba"][0] * 255)
    codes = torch.from_numpy(host[M - 1]).to(dev())
    v = _views(M - 1, M, (0,))
    a = lambda x, dt=np.float32: np.ascontiguousarray(x, dtype=dt)
    keep = dict(view2mpi=a(v["view2mpi"], np.int32), dhw=a(v["dhw"]), ray_dir=a(v["ray_dir"]), eye=a(v["eye"]), z_dir=a(v["z_dir"]),
                color=np.empty((1, 3, R, R), np.float32), depth=np.empty((1, 1, R, R), np.float32), flags=np.zeros(1, np.uint32))
    desc = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | _lib.OPT_MPI_U8, M=M, V=1, N=N, Ht=R, Wt=R, H=R,
                          W=R, rgba=host.ctypes.data, **{k: x.ctypes.data for k, x in keep.items()})
    lib = _lib.load()
    torch.cuda.synchronize()
    free = torch.cuda.mem_get_info()[0]
    try:
        _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(desc), torch.cuda.current_device()))
        # the library's staging slots are its own cudaMalloc, which torch's peak (the budget fixture) does not see
        staging = free - torch.cuda.mem_get_info()[0]
    finally:
        _lib.check(lib.gmpi_mpi_release_host_cache())
    print("LARGE_OFFSETS_HOST_STAGING " + json.dumps(dict(staging_gb=round(staging / 1e9, 2))))
    del host
    ref = render_fwd(_views(0, 1, (0,)), {"rgba": codes[None]})
    assert_bitwise((keep["color"], keep["depth"], keep["flags"].view(np.int32)), ref, "host != device")


# ------------------------------------------------------------------------------------------------------------------------------
# the benchmark's batch: FFHQ1024, 4 MPIs of 96 x 1024^2 in one 6.4 GB tensor (MPI 2 starts past 2^31 bytes, MPI 3 past 2^32)
# ------------------------------------------------------------------------------------------------------------------------------
def test_the_benchmark_batch_of_four(budget):
    """At its automatic kernel choice (the staged kernel on its 2-stage ring): each view k is bitwise the render of MPI k copied
    alone into a fresh allocation; the fp16 and uint8 renders are bitwise those of their fp32 conversions; the factored render is
    bitwise its expanded form's; skip_empty is bitwise the plain render."""
    budget("batch_of_four")
    set_kernel("auto")
    d = dev()
    assert _ring_kernel(4, 4) == "staged2"
    geo = synth.make_case(n_planes=N, tex=8, img=R, n_mpi=4, seed=1234, rgba=False)
    c = dict(view2mpi=geo.view2mpi.numpy(), dhw=geo.dhw.numpy(), ray_dir=geo.ray_dir.numpy(), eye=geo.eye.numpy(), z_dir=geo.z_dir.numpy(),
             ac=True)
    gen = torch.Generator(device=d).manual_seed(5)
    rgba = torch.rand((4, N, 4, R, R), generator=gen, device=d)
    rgba[:, :, 3] = synth.equal_weight_alpha((4, N, R, R), gen, d)
    base = render_fwd(c, {"rgba": rgba})
    for k in range(4):
        ck = dict(c, view2mpi=np.zeros(1, np.int32), dhw=c["dhw"][k:k + 1], ray_dir=c["ray_dir"][k:k + 1], eye=c["eye"][k:k + 1],
                  z_dir=c["z_dir"][k:k + 1])
        assert _ring_kernel(1, 1) == "staged2"
        alone = render_fwd(ck, {"rgba": rgba[k:k + 1].clone()})
        assert_bitwise((base[0][k], base[1][k]), (alone[0][0], alone[1][0]), ("view", k))
    t = lambda a: torch.from_numpy(a).to(d)
    args = (t(c["dhw"]), t(c["view2mpi"]), t(c["ray_dir"]), t(c["eye"]), t(c["z_dir"]))
    plain = g.render_views(rgba, *args)
    assert_bitwise(g.render_views(rgba, *args, skip_empty=True), plain, "skip_empty != plain")
    del plain
    rgb, bg = torch.rand((4, 3, R, R), generator=gen, device=d), torch.rand((4, 3, R, R), generator=gen, device=d)
    alpha = rgba[:, :, 3:4].clone()
    rgba[:, :, :3] = rgb[:, None]           # rgba becomes the expanded form (expand_factored, without its temporaries)
    rgba[:, -1, :3] = bg
    assert_bitwise(render_fwd(c, dict(rgb=rgb, alpha=alpha, bg_rgb=bg)), render_fwd(c, {"rgba": rgba}), "factored != expanded")
    del alpha, rgb, bg
    half = rgba.half()
    del rgba
    up = half.float()
    h, f, fell_back = native_vs_fp32(c, {"rgba": half}, {"rgba": up}, "auto")
    assert not fell_back
    assert_bitwise(h, f, "fp16 != its upcast")
    del half
    codes = up.mul_(255).round_().to(torch.uint8)
    del up
    conv = _unorm8_conversion(codes)
    h, f, fell_back = native_vs_fp32(c, {"rgba": codes}, {"rgba": conv}, "auto")
    assert not fell_back
    assert_bitwise(h, f, "uint8 != its conversion")
