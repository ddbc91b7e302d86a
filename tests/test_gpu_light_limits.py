"""LightRenderer's kernels (csrc/mpi_light.cuh, through ml_gmpi_b200/light.py) against a float64 restatement of the two operations
they compute, at the shapes, layouts and alpha values where a streaming kernel goes wrong (run on an H100: pytest -m gpu).

  compute_depth  s_i = 1 - a_i + 1e-10,  T_i = prod_{j<i} s_j,  depth = sum_i a_i T_i d_i   (a_i: the fp32 alpha cast to fp64);
                 d depth / d alpha from fp64 autograd of that formula.
  shading        clip(rgb * s, 0, 1) on the colour channels, alpha passed through.

Shapes: a ragged second block (20x52 texels = 260 four-texel threads), a float4 spanning two rows (6x10), the training shape
(4 MPIs x 32 planes x 256^2, FFHQ plane distances), 17 MPIs, 1 and 512 planes, the benchmark's 4 x 96 x 1024^2, and the odd
texel counts 33x33 and 5x7, which the kernels do not stream and light.py computes with fp32 torch.  Alpha patterns (64^2, 16
planes): all 0, all 1, plane 0 = 1, 3 and 6 consecutive planes = 1 mid-stack (T runs through fp32 subnormals into 0), exactly 0.5,
random with the last plane = 1.  Every case but the patterns has its last plane at alpha = 1, as the generator's MPIs do.

Bars (u = 2^-24; derived from the arithmetic, not fitted):
  depth    |err| <= (4N+4) u sum_i a_i T_i d_i + N 2^-126 max d.
           Every term of the sum is non-negative, so relative errors of terms add.  The kernel's factor fl(fl(1 - a) + 1e-10f) is
           s_i (1 + 2u) at worst: 1 - a rounds by u, 1e-10f differs from 1e-10 by u of 1e-10 <= u s_i, the sum rounds by u.  Each
           product of T adds u, so T_i carries 3i u; a_i T_i rounds once, and the fma chain rounds the running sum N - i times once
           term i is in: (3i + 1 + N - i) u <= (3N - 1) u.  The odd sizes' torch expression (cumprod, a*T and *d as two products, a
           reduction over N planes) reaches (4N - 3) u, so one bar with room for the second-order terms covers both.  Once T is
           subnormal a product rounds by up to 2^-150 absolutely; over N planes that stays far below the N 2^-126 max d floor.
  d alpha  g_i = T_i G (d_i - R_i),  R_i = sum_{j>i} a_j d_j prod_{i<k<j} s_k  (the kernel's back-to-front recurrence, times G).
           |err_i| <= (4N+4) u T_i |G| (d_i + R_i) + N 2^-126 (|G| (d_i + R_i) + 1).
           Term j of R_i carries 4 (j - i) - 2 roundings: G d_j, its fma, and per plane k in between 2 in s_k, the product and the
           fma.  With T_i's 3i, the difference and the last product: 3i + 4 (j - i) <= 4N - 4; the d_i term carries 3i + 3 <= 3N.
           The torch expression's autograd (cumprod's backward divides a reversed cumulative sum by s_i) reaches (4N + 3) u while T
           stays normal; divided by s_i = 1e-10 (alpha = 1) a subnormal T's rounding is magnified 1e10 times, which is why the
           kernel's backward does not divide and why the odd sizes, which take that expression, are tested with random alpha only.
           The bar is absolute in T_i |G| (d_i + R_i), never relative to g_i, so the cancellation between d_i and R_i cannot break
           it.  The floor covers subnormal T and R.
  shading  The forward and d rgb are bit for bit the fp32 torch expression cat(clip(rgb * s, 0, 1), alpha) and its autograd, with
           NaN positions matched as sets (every element is one rounding of the same product, and the same masked product; with
           rgb and alpha split apart, so that autograd adds no zero fill that would turn a -0 gradient into +0);
           d alpha is bit for bit g_out[:, :, 3].  d s against the fp64 sum of mask * g * rgb, the mask taken from the fp32 product
           (the closed interval decides at exactly 0 and 1): the kernel sums 3N exact products with one rounding each, so
           |err| <= 3N u sum |mask g rgb| + 3N 2^-149, and NaN positions are equal.
LightRenderer.render end to end is held to twice the error of the same method in fp32 torch, both against fp64.
test_the_bars_fail_on_slightly_wrong_problems shows that every check above rejects a plausible mistake by a wide margin."""
import json

import pytest
import torch

from ml_gmpi_b200 import light
from ml_gmpi_b200.geometry import FFHQ, plane_dhw_table, texel_xyzd
from ml_gmpi_b200.light import LightRenderer, alpha_depth, apply_shading
from testlib import dev

pytestmark = pytest.mark.gpu
U = 2.0 ** -24
MIN_NORMAL = 2.0 ** -126
MIN_SUBNORMAL = 2.0 ** -149


def report(tag, **kw):
    print(tag + " " + json.dumps({k: (float("%.3g" % v) if isinstance(v, float) else v) for k, v in kw.items()}))


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------
def ffhq_dhw(n):
    """[n, 3] (distance, height, width) of the FFHQ configuration's planes, fp32 on the device."""
    return torch.from_numpy(plane_dhw_table(n_planes=n, **FFHQ)).to(dev())


PATTERNS = ["zeros", "ones", "plane0_one", "three_ones_mid", "six_ones_mid", "half", "random_last_one"]


def make_alpha(M, N, H, W, pattern="random_last_one", seed=0):
    gen = torch.Generator(device=dev()).manual_seed(seed)
    a = torch.rand((M, N, 1, H, W), generator=gen, device=dev())
    if pattern == "zeros":
        a.zero_()
    elif pattern == "ones":
        a.fill_(1.0)
    elif pattern == "plane0_one":
        a[:, 0] = 1.0
    elif pattern == "three_ones_mid":
        a[:, 5:8] = 1.0                          # T = 1e-30 behind them: still normal in fp32
    elif pattern == "six_ones_mid":
        a[:, 5:11] = 1.0                         # 1e-40 (subnormal), then 0 in fp32; the fp64 reference keeps 1e-60
    elif pattern == "half":
        a.fill_(0.5)
    else:
        assert pattern == "random_last_one", pattern
        a[:, -1] = 1.0
    return a


def make_shading(M, N, H, W, seed=0, nonfinite=False):
    """rgba [M,N,4,H,W], shade [M,1,H,W] and g_out.  Colours in [-0.25, 1.25] and shades in [0, 1.6] put products below 0, inside
    and above 1; a share of the elements take the clip's edge values: rgb 0.5 with shade 2 (product exactly 1), rgb 0, -0.0 and 1,
    the next float above 1, shade 0 and 1 -- and with `nonfinite` also rgb NaN and +-inf, shade NaN and inf (inf * 0 = NaN).
    The alpha channel takes the same values: it must pass through bit for bit."""
    gen = torch.Generator(device=dev()).manual_seed(1000 + seed)
    rgba = torch.rand((M, N, 4, H, W), generator=gen, device=dev()) * 1.5 - 0.25
    shade = torch.rand((M, 1, H, W), generator=gen, device=dev()) * 1.6
    g_out = torch.randn((M, N, 4, H, W), generator=gen, device=dev())
    above_one = 1.0 + 2.0 ** -23
    rgb_specials = [(0.5, 0.04), (0.0, 0.02), (-0.0, 0.02), (1.0, 0.02), (above_one, 0.02)]
    shade_specials = [(2.0, 0.08), (0.0, 0.05), (1.0, 0.05)]
    if nonfinite:
        rgb_specials += [(float("nan"), 0.01), (float("inf"), 0.01), (float("-inf"), 0.005)]
        shade_specials += [(float("nan"), 0.03), (float("inf"), 0.03)]
    for t, specials in ((rgba, rgb_specials), (shade, shade_specials)):
        flat = t.view(-1)
        for lo in range(0, flat.numel(), 1 << 26):               # bounded temporaries at the benchmark's size
            part = flat[lo:lo + (1 << 26)]
            r = torch.rand(part.shape, generator=gen, device=dev())
            acc = 0.0
            for v, p in specials:
                part.masked_fill_((r >= acc) & (r < acc + p), v)
                acc += p
    return rgba, shade, g_out


# ------------------------------------------------------------------------------------------------------------------------------
# compute_depth: kernel runs, fp64 reference, bars
# ------------------------------------------------------------------------------------------------------------------------------
def depth_kernel(alpha, d, G):
    """The kernel's depth with T stored, its d alpha for the upstream gradient G, and the depth of the forward without T."""
    leaf = alpha.clone().requires_grad_(True)
    depth = alpha_depth(leaf, d)
    depth.backward(G)
    depth_no_t = alpha_depth(alpha, d)
    return depth.detach(), leaf.grad, depth_no_t


DEPTH_WRONG = ["d_shifted", "t_inclusive", "mpi_off_by_one"]


def depth_errors(alpha, d, G, depth_k, g_k, wrong=None):
    """max |err| / bar of the depth and of d alpha against the fp64 reference, built one MPI at a time to bound memory.  `wrong`
    makes the reference that of a slightly wrong problem: each plane weighted with the next plane's distance, T_i including plane
    i, or MPI m computed from MPI m+1's alpha."""
    M, N = alpha.shape[:2]
    dv = d.double().reshape(N, 1, 1)
    if wrong == "d_shifted":
        dv = torch.cat((dv[1:], dv[-1:]))
    worst = dict(depth=0.0, g_alpha=0.0)
    for m in range(M):
        src = (m + 1) % M if wrong == "mpi_off_by_one" else m
        a = alpha[src, :, 0].double().requires_grad_(True)
        s = 1.0 - a + 1e-10
        T = torch.cumprod(s if wrong == "t_inclusive" else torch.cat((torch.ones_like(s[:1]), s[:-1])), dim=0)
        depth = (a * T * dv).sum(0)
        Gm = G[m, 0].double()
        g, = torch.autograd.grad(depth, a, Gm)
        with torch.no_grad():
            R = torch.zeros_like(a)
            for i in range(N - 2, -1, -1):
                R[i] = a[i + 1] * dv[i + 1] + s[i + 1] * R[i + 1]
            bar_d = (4 * N + 4) * U * depth + N * MIN_NORMAL * float(dv.max())
            scale = Gm.abs() * (dv + R)
            bar_g = (4 * N + 4) * U * T.detach() * scale + N * MIN_NORMAL * (scale + 1.0)
            worst["depth"] = max(worst["depth"], float(((depth_k[m, 0].double() - depth) / bar_d).abs().max()))
            worst["g_alpha"] = max(worst["g_alpha"], float(((g_k[m, :, 0].double() - g) / bar_g).abs().max()))
    return worst


def check_depth(alpha, d, label):
    gen = torch.Generator(device=dev()).manual_seed(7)
    G = torch.randn((alpha.shape[0], 1) + alpha.shape[-2:], generator=gen, device=dev())
    depth_k, g_k, depth_no_t = depth_kernel(alpha, d, G)
    assert torch.equal(depth_k.view(torch.int32), depth_no_t.view(torch.int32)), label
    assert g_k.shape == alpha.shape and g_k.dtype == torch.float32
    e = depth_errors(alpha, d, G, depth_k, g_k)
    report("LIGHT_DEPTH", case=label, **e)
    assert max(e.values()) <= 1.0, (label, e)
    return e


# ------------------------------------------------------------------------------------------------------------------------------
# apply_shading: bitwise against fp32 torch, d shade against fp64
# ------------------------------------------------------------------------------------------------------------------------------
def shading_expr(rgba, shade, open_at_one=False):
    """The fp32 torch expression apply_shading replaces, on rgba [M,N,4,H,W] and shade [M,1,H,W].  `open_at_one`: the same values,
    with the gradient cut at exactly 1 (a slightly wrong problem: torch.clip passes the gradient on the closed interval).
    rgb and alpha come from split, whose backward concatenates their gradients: taken as two slices, autograd would add each
    slice's gradient to the other's zero fill, and -0 + 0 turns d rgb = g * 0 with g < 0 into +0 where the kernel writes g * s."""
    rgb, alpha = rgba.split((3, 1), dim=2)
    p = rgb * shade.unsqueeze(1)
    c = torch.where(p >= 1, torch.ones_like(p), torch.clip(p, min=0.0)) if open_at_one else torch.clip(p, min=0.0, max=1.0)
    return torch.cat((c, alpha), dim=2)


def bit_mismatches(x, y):
    """Elements whose bit patterns differ, NaN positions compared as sets (a NaN's payload is not)."""
    nx, ny = torch.isnan(x), torch.isnan(y)
    both = ~(nx | ny)
    return int((nx != ny).sum()) + int(((x.view(torch.int32) != y.view(torch.int32)) & both).sum())


SHADING_WRONG = ["clip_open_at_one", "g_shade_n_minus_1", "mpi_off_by_one"]


def shading_errors(rgba, shade, g_out, wrongs=(None,)):
    """Per entry of `wrongs` (None: the right problem): mismatched bits of the forward, of d rgb and of d alpha, unequal NaN
    positions of d shade and max |err| / bar of d shade, against the reference of that problem.  The kernel's forward is freed
    before its backward runs, and the references are built one MPI at a time, to bound memory at the benchmark's size."""
    M, N = rgba.shape[:2]
    res = {w: dict(fwd_bits=0, g_rgb_bits=0, g_alpha_bits=0, g_shade_nan=0, g_shade=0.0) for w in wrongs}
    src = lambda w, m: (m + 1) % M if w == "mpi_off_by_one" else m
    with torch.no_grad():
        out = apply_shading(rgba, shade)
        for w in wrongs:
            for m in range(M):
                j = src(w, m)
                res[w]["fwd_bits"] += bit_mismatches(out[m:m + 1], shading_expr(rgba[j:j + 1], shade[j:j + 1], w == "clip_open_at_one"))
    del out
    x, s = rgba.requires_grad_(True), shade.clone().requires_grad_(True)
    apply_shading(x, s).backward(g_out)
    g_rgba, g_shade = x.grad, s.grad
    x.requires_grad_(False)
    x.grad = None
    assert g_rgba.shape == rgba.shape and g_shade.shape == shade.shape
    for w in wrongs:
        r = res[w]
        for m in range(M):
            j = src(w, m)
            xr = rgba[j:j + 1].clone().requires_grad_(True)
            shading_expr(xr, shade[j:j + 1], w == "clip_open_at_one").backward(g_out[m:m + 1])
            r["g_rgb_bits"] += bit_mismatches(g_rgba[m, :, :3], xr.grad[0, :, :3])
            r["g_alpha_bits"] += bit_mismatches(g_rgba[m, :, 3], g_out[m, :, 3])
            del xr
            with torch.no_grad():
                rgb = rgba[j, :, :3]
                p = rgb * shade[j]
                mask = (p >= 0) & ((p < 1) if w == "clip_open_at_one" else (p <= 1))
                terms = mask.double() * g_out[m, :, :3].double() * rgb.double()
                if w == "g_shade_n_minus_1":
                    terms = terms[:-1]
                ref = terms.sum((0, 1))
                bar = 3 * N * U * terms.abs().sum((0, 1)) + 3 * N * MIN_SUBNORMAL
                del terms, mask, p
                k = g_shade[m, 0].double()
                nk, nr = torch.isnan(k), torch.isnan(ref)
                r["g_shade_nan"] += int((nk != nr).sum())
                ok = ~(nk | nr)
                if bool(ok.any()):
                    r["g_shade"] = max(r["g_shade"], float(((k - ref).abs() / bar)[ok].max()))
    return res


def check_shading(rgba, shade, g_out, label):
    e = shading_errors(rgba, shade, g_out)[None]
    report("LIGHT_SHADING", case=label, **e)
    assert e["fwd_bits"] == 0 and e["g_rgb_bits"] == 0 and e["g_alpha_bits"] == 0 and e["g_shade_nan"] == 0, (label, e)
    assert e["g_shade"] <= 1.0, (label, e)
    return e


# ------------------------------------------------------------------------------------------------------------------------------
# 1. shapes and alpha patterns
# ------------------------------------------------------------------------------------------------------------------------------
SHAPES = {                                 # M, N, Ht, Wt
    "ragged_block_20x52": (3, 8, 20, 52),  # 260 four-texel threads: a second block with 4 live threads
    "float4_spans_rows_6x10": (2, 8, 6, 10),
    "training_4x32x256": (4, 32, 256, 256),
    "many_mpis_17x8x64": (17, 8, 64, 64),
    "one_plane_64": (2, 1, 64, 64),
    "planes_512_64": (2, 512, 64, 64),
    "odd_33x33": (2, 8, 33, 33),
    "odd_5x7": (3, 4, 5, 7),
    "benchmark_4x96x1024": (4, 96, 1024, 1024),
}


@pytest.mark.parametrize("name", list(SHAPES))
def test_compute_depth_and_its_gradient_against_float64(name):
    M, N, H, W = SHAPES[name]
    check_depth(make_alpha(M, N, H, W, seed=N), ffhq_dhw(N)[:, 0].contiguous(), name)


@pytest.mark.parametrize("pattern", PATTERNS)
def test_compute_depth_alpha_patterns_against_float64(pattern):
    check_depth(make_alpha(2, 16, 64, 64, pattern, seed=3), ffhq_dhw(16)[:, 0].contiguous(), pattern)


@pytest.mark.parametrize("name", list(SHAPES))
def test_apply_shading_against_torch_and_float64(name):
    M, N, H, W = SHAPES[name]
    check_shading(*make_shading(M, N, H, W, seed=N), name)


@pytest.mark.parametrize("shape", [(3, 4, 20, 52), (4, 16, 6, 10), (4, 32, 5, 7)], ids=["20x52", "6x10", "odd_5x7"])
def test_apply_shading_keeps_nan_and_every_clip_edge_as_torch(shape):
    """NaN colours, NaN shades and inf * 0 stay NaN as with torch.clip (which keeps NaN where fmaxf would return 0), products of
    exactly 0 and 1, -0.0 and the next float above 1 clip as torch clips them, and the gradient's mask and d shade follow."""
    rgba, shade, g_out = make_shading(*shape, seed=11, nonfinite=True)
    p = rgba[:, :, :3] * shade.unsqueeze(1)
    assert int((p == 1).sum()) and int((p == 0).sum()) and int(torch.isnan(p).sum())
    assert int(((rgba[:, :, :3] == 0) & torch.signbit(rgba[:, :, :3])).sum()) and int((p == 1.0 + 2.0 ** -23).sum())
    assert int((torch.isinf(rgba[:, :, :3]) & (shade.unsqueeze(1) == 0)).sum()) and int(torch.isnan(shade).sum())
    out = apply_shading(rgba, shade)
    assert int(torch.isnan(out[:, :, :3]).sum()) == int(torch.isnan(p).sum())
    check_shading(rgba, shade, g_out, "edges_%dx%d" % shape[2:])


# ------------------------------------------------------------------------------------------------------------------------------
# 2. layouts: what _alpha_view reads in place and what it copies give the same bits
# ------------------------------------------------------------------------------------------------------------------------------
def test_alpha_layouts_give_the_contiguous_result_bit_for_bit():
    """At 256^2 with a gradient: the channel-3 view of an [M,N,4,H,W] stack and every other plane are read in place, a transposed
    H/W view and a base offset by one float are copied (the offset one is contiguous, so only its alignment tells that it must
    be), fp16 alpha is upcast; plane distances come as [N], [N,1] or fp64.  Each
    gives the contiguous fp32 result bit for bit, its gradient lands where its alpha came from, and nothing else is written."""
    M, N, H, W = 2, 8, 256, 256
    d = ffhq_dhw(N)[:, 0].contiguous()
    base = make_alpha(M, N, H, W, seed=5)
    G = torch.randn((M, 1, H, W), generator=torch.Generator(device=dev()).manual_seed(9), device=dev())
    bits = lambda t: t.detach().contiguous().view(torch.int32)

    def run(leaf, view_of, plane_ds=d):
        depth = alpha_depth(view_of(leaf), plane_ds)
        depth.backward(G)
        return depth.detach(), leaf.grad

    depth_c, g_c = run(base.clone().requires_grad_(True), lambda t: t)
    check = depth_errors(base, d, G, depth_c, g_c)
    assert max(check.values()) <= 1.0, check

    stack = torch.randn((M, N, 4, H, W), device=dev())
    stack[:, :, 3:] = base
    stack.requires_grad_(True)
    depth, g = run(stack, lambda t: t[:, :, 3:])
    assert torch.equal(bits(depth), bits(depth_c)) and torch.equal(bits(g[:, :, 3:]), bits(g_c))
    assert torch.equal(bits(g[:, :, :3]), torch.zeros_like(bits(g[:, :, :3])))

    every_other = torch.zeros((M, 2 * N, 1, H, W), device=dev())
    every_other[:, ::2] = base
    depth, g = run(every_other.requires_grad_(True), lambda t: t[:, ::2])
    assert torch.equal(bits(depth), bits(depth_c)) and torch.equal(bits(g[:, ::2]), bits(g_c))
    assert torch.equal(bits(g[:, 1::2]), torch.zeros_like(bits(g[:, 1::2])))

    depth, g = run(base.transpose(-1, -2).contiguous().requires_grad_(True), lambda t: t.transpose(-1, -2))
    assert torch.equal(bits(depth), bits(depth_c)) and torch.equal(bits(g.transpose(-1, -2)), bits(g_c))

    flat = torch.zeros(base.numel() + 1, device=dev())
    flat[1:] = base.reshape(-1)
    depth, g = run(flat.requires_grad_(True), lambda t: t[1:].view(M, N, 1, H, W))
    assert torch.equal(bits(depth), bits(depth_c)) and torch.equal(bits(g[1:]), bits(g_c).reshape(-1)) and float(g[0]) == 0.0

    half = base.half()
    depth32, g32 = run(half.float().requires_grad_(True), lambda t: t)
    depth, g = run(half.clone().requires_grad_(True), lambda t: t)
    assert g.dtype == torch.float16 and torch.equal(bits(depth), bits(depth32))
    assert torch.equal(g.view(torch.int16), g32.half().view(torch.int16))

    for pd in (d.reshape(N, 1), d.double()):
        depth, g = run(base.clone().requires_grad_(True), lambda t: t, pd)
        assert torch.equal(bits(depth), bits(depth_c)) and torch.equal(bits(g), bits(g_c)), (pd.shape, pd.dtype)


def test_apply_shading_copies_an_unaligned_stack():
    """An MPI and a shading that start one float into their allocations cannot be read as float4s: they are copied, and the
    shaded MPI and both gradients are bit for bit those of aligned tensors."""
    rgba, shade, g_out = make_shading(2, 4, 20, 52, seed=3)
    x, s = rgba.clone().requires_grad_(True), shade.clone().requires_grad_(True)
    out = apply_shading(x, s)
    out.backward(g_out)

    def offset(t):
        flat = torch.zeros(t.numel() + 1, device=dev())
        flat[1:] = t.reshape(-1)
        return flat.requires_grad_(True)

    fx, fs = offset(rgba), offset(shade)
    out_u = apply_shading(fx[1:].view(rgba.shape), fs[1:].view(shade.shape))
    out_u.backward(g_out)
    assert bit_mismatches(out_u, out) == 0
    assert bit_mismatches(fx.grad[1:], x.grad.reshape(-1)) == 0 and bit_mismatches(fs.grad[1:], s.grad.reshape(-1)) == 0
    assert float(fx.grad[0]) == 0.0 and float(fs.grad[0]) == 0.0


def test_no_grad_forward_allocates_only_the_depth():
    """T (4 B per texel-plane) is what the backward reads: under torch.no_grad a grad-requiring alpha must not allocate it; with
    grad it is stored (which shows that the measurement sees it)."""
    M, N, H, W = 4, 96, 256, 256
    a = make_alpha(M, N, H, W).requires_grad_(True)
    d = ffhq_dhw(N)[:, 0].contiguous()
    depth_bytes, t_bytes = M * H * W * 4, M * N * H * W * 4

    def peak_of(fn):
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        before = torch.cuda.memory_allocated()
        out = fn()
        torch.cuda.synchronize()
        return out, torch.cuda.max_memory_allocated() - before

    with torch.no_grad():
        depth, extra = peak_of(lambda: alpha_depth(a, d))
    assert extra == depth_bytes, (extra, depth_bytes)
    del depth
    depth, extra = peak_of(lambda: alpha_depth(a, d))
    assert extra >= depth_bytes + t_bytes, (extra, depth_bytes + t_bytes)


# ------------------------------------------------------------------------------------------------------------------------------
# 3. LightRenderer.render end to end
# ------------------------------------------------------------------------------------------------------------------------------
def depth_torch(mpi_alpha, plane_ds):
    """compute_depth restated in torch, in the dtype of its input."""
    a = mpi_alpha[:, :, 0]
    s = (1.0 - a) + 1e-10
    T = torch.cumprod(torch.cat((torch.ones_like(s[:, :1]), s[:, :-1]), dim=1), dim=1)
    return (a * T * plane_ds.reshape(1, -1, 1, 1).to(a.dtype)).sum(1, keepdim=True)


def shading_torch(batch_mpi, shading):
    B, N, _, H, W = batch_mpi.shape
    return shading_expr(batch_mpi, shading.reshape(B, 1, H, W))


def test_light_render_end_to_end_is_as_accurate_as_fp32_torch(monkeypatch):
    """render forward and backward at the training shape with a fixed light: its error against the same method run in fp64 is at
    most twice the error of the method run in fp32 torch (the reference's own arithmetic), plus 8 u of the output's scale.  The
    colours stay in [0.02, 0.7] so that no product reaches a clip edge and the three runs share one gradient mask; g_out's
    alpha channel is 0 so that d alpha is what flows back through the shading, the normals, the blur and compute_depth."""
    M, N, H, W = 4, 32, 256, 256
    gen = torch.Generator(device=dev()).manual_seed(21)
    dhw = ffhq_dhw(N)
    xyz = texel_xyzd(dhw, H, W)
    rgb = 0.02 + 0.68 * torch.rand((M, N, 3, H, W), generator=gen, device=dev())
    mpi = torch.cat((rgb, make_alpha(M, N, H, W, seed=4)), dim=2)
    g_out = torch.randn(mpi.shape, generator=gen, device=dev())
    g_out[:, :, 3] = 0.0
    yaws, pitches = torch.tensor([[0.3], [-0.2], [0.1], [-0.05]]), torch.tensor([[0.1], [0.15], [-0.1], [0.05]])
    monkeypatch.setattr(torch.backends.cudnn, "allow_tf32", False)    # the blur is a convolution: keep it fp32 in every run

    def run(dtype):
        lr = LightRenderer(sphere_center_z=1.0, sphere_r=1.0, ka_max=0.7, kd_max=0.6, n_grow_iters=10)
        lr.step = 20
        x = mpi.to(dtype, copy=True).requires_grad_(True)
        out = lr.render(x, dhw.to(dtype), xyz.to(dtype), given_yaws=yaws, given_pitches=pitches)
        out.backward(g_out.to(dtype))
        return dict(out=out.detach().double(), g_rgb=x.grad[:, :, :3].double(), g_alpha=x.grad[:, :, 3].double())

    ours = run(torch.float32)
    with monkeypatch.context() as mp:
        mp.setattr(light, "alpha_depth", depth_torch)
        mp.setattr(light, "apply_shading", shading_torch)
        exact, fp32 = run(torch.float64), run(torch.float32)
    for k in ours:
        scale = float(exact[k].abs().max())
        e_ours = float((ours[k] - exact[k]).abs().max()) / scale
        e_fp32 = float((fp32[k] - exact[k]).abs().max()) / scale
        report("LIGHT_RENDER", output=k, err=e_ours, err_fp32_torch=e_fp32, ratio=e_ours / max(e_fp32, 1e-30))
        assert e_ours <= 2 * e_fp32 + 8 * U, (k, e_ours, e_fp32)


# ------------------------------------------------------------------------------------------------------------------------------
# 4. the bars have teeth
# ------------------------------------------------------------------------------------------------------------------------------
def test_the_bars_fail_on_slightly_wrong_problems():
    """The kernels' results on the right problem, checked with the same helpers against the reference of a slightly wrong one:
    the depth with the next plane's distance, an inclusive T, the next MPI's alpha; the shading with the gradient cut at exactly 1,
    d shade summed over N - 1 planes, the next MPI's data.  Each must fail its bars by 10x or more (a bitwise check: by one
    element or more)."""
    M, N, H, W = 3, 16, 64, 64
    alpha, d = make_alpha(M, N, H, W, seed=2), ffhq_dhw(N)[:, 0].contiguous()
    G = torch.randn((M, 1, H, W), generator=torch.Generator(device=dev()).manual_seed(8), device=dev())
    depth_k, g_k, _ = depth_kernel(alpha, d, G)
    assert max(depth_errors(alpha, d, G, depth_k, g_k).values()) <= 1.0
    for wrong in DEPTH_WRONG:
        e = depth_errors(alpha, d, G, depth_k, g_k, wrong)
        report("LIGHT_TEETH", wrong="depth_" + wrong, **e)
        assert max(e.values()) >= 10, (wrong, e)

    res = shading_errors(*make_shading(3, 4, 20, 52, seed=11, nonfinite=True), wrongs=[None] + SHADING_WRONG)
    assert res[None]["g_shade"] <= 1.0 and sum(v for k, v in res[None].items() if k != "g_shade") == 0, res[None]
    for wrong in SHADING_WRONG:
        e = res[wrong]
        report("LIGHT_TEETH", wrong="shading_" + wrong, **e)
        assert e["g_shade"] >= 10 or e["fwd_bits"] + e["g_rgb_bits"] + e["g_shade_nan"] > 0, (wrong, e)
