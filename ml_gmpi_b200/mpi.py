"""Drop-in for `gmpi.core.mpi.MPI` (reference gmpi/core/mpi.py:156-436), backed by the sm_90a
kernels through the C ABI.  Same constructor, same keyword-only `forward`, same return values,
same assertion messages; differentiable w.r.t. `batch_rgba` (first order), which is all the
reference's callers need (the sampling grid and the depth are built under no_grad,
mpi.py:65,148).

No CPU path: tensors must live on a CUDA device, otherwise this raises.
"""
import ctypes
import warnings
from typing import List, NamedTuple, Optional, Tuple, Union

import numpy as np
import torch
from torch import nn

from . import _lib


class MPIOutOfPlaneError(AssertionError):
    """Rays leave the last plane (reference: prints the poses and sys.exit(1), mpi.py:103-128)."""


def _stream_ptr(device):
    return torch.cuda.current_stream(device).cuda_stream


def _require_cuda(t: torch.Tensor, who: str = "ml_gmpi_b200 renders"):
    if not t.is_cuda:
        raise RuntimeError(f"{who} on CUDA devices only (no CPU fallback); got a CPU tensor")


def _zero_flags(device) -> torch.Tensor:
    return torch.zeros(1, dtype=torch.int32, device=device)


def _as_f32c(t: torch.Tensor) -> torch.Tensor:
    if t.dtype != torch.float32:
        t = t.float()
    return t if t.is_contiguous() else t.contiguous()


class _RenderFn(torch.autograd.Function):
    """MPI.forward + its autograd through the C ABI's descriptor entry points (gmpi_mpi_render_fwd_ex / _bwd_ex).
    The MPI is either expanded (`rgba`) or factored (`rgb`, `alpha`, optional `bg_rgb`); the unused form is None."""

    @staticmethod
    def forward(ctx, rgba, rgb, alpha, bg_rgb, dhw, view2mpi, ray_dir, eye, z_dir, options, flags, view_group, early_stop,
                deterministic, occ=None):
        mpi = [rgba, rgb, alpha, bg_rgb]
        V, _, H, W = ray_dir.shape
        ref = _mpi_ref(mpi)
        dev = ref.device
        color = torch.empty((V, 3, H, W), device=dev, dtype=torch.float32)
        depth = torch.empty((V, 1, H, W), device=dev, dtype=torch.float32)
        # training: the forward also saves the transmittance in front of every plane (4 B per pixel-plane) so that the
        # backward is ONE staged back-to-front sweep (torch autograd keeps ~30 such tensors alive for the reference)
        trans = None
        if any(ctx.needs_input_grad[:4]):
            trans = torch.empty((V, ref.shape[1], H, W), device=dev, dtype=torch.float32)
        _render_fwd(_mpi_desc(mpi, V, H, W, options, view_group=view_group, view2mpi=view2mpi, dhw=dhw, ray_dir=ray_dir, eye=eye,
                              z_dir=z_dir, color=color, depth=depth, transmittance=trans, flags=flags, early_stop=early_stop),
                    occ, dev)
        ctx.save_for_backward(rgba, rgb, alpha, bg_rgb, dhw, view2mpi, ray_dir, eye, z_dir, trans)
        ctx.options, ctx.view_group = options, view_group
        # None: torch's global switch, read now (the backward may run on an autograd thread, after the caller changed it)
        ctx.deterministic = torch.are_deterministic_algorithms_enabled() if deterministic is None else bool(deterministic)
        ctx.set_materialize_grads(False)
        return color, depth

    @staticmethod
    @torch.autograd.function.once_differentiable     # raw kernels: a double backward (create_graph=True) must raise, not
    def backward(ctx, g_color, g_depth):             # silently treat the result as constant (the reference's R1 only differentiates D)
        rgba, rgb, alpha, bg_rgb, dhw, view2mpi, ray_dir, eye, z_dir, trans = ctx.saved_tensors
        none = (None,) * 15
        if not any(ctx.needs_input_grad[:4]):
            return none
        lib = _lib.load()
        mpi = [rgba, rgb, alpha, bg_rgb]
        V, _, H, W = ray_dir.shape
        dev = _mpi_ref(mpi).device
        if g_color is None:
            g_color = torch.zeros((V, 3, H, W), device=dev, dtype=torch.float32)
        g_color = _as_f32c(g_color)
        g_depth = _as_f32c(g_depth) if g_depth is not None else None
        # GMPI_ZERO_GRAD: the callee zeroes the buffers on the stream.  (Zeroing them on a side stream during the forward, as an
        # earlier version did, buys nothing: a memset cannot overlap the persistent kernels -- tools/zero_overlap_probe.py.)
        if rgba is None:
            g_rgba = None
            g_rgb, g_alpha = torch.empty_like(rgb), torch.empty_like(alpha)
            g_bg = torch.empty_like(bg_rgb) if bg_rgb is not None else None
        else:
            g_rgb = g_alpha = g_bg = None
            g_rgba = torch.empty_like(rgba)
        with torch.cuda.device(dev):   # autograd worker threads do not inherit the device
            d = _mpi_desc(mpi, V, H, W, ctx.options | _lib.OPT_ZERO_GRAD, view_group=ctx.view_group, view2mpi=view2mpi, dhw=dhw,
                          ray_dir=ray_dir, eye=eye, z_dir=z_dir, transmittance=trans, g_color=g_color, g_depth=g_depth,
                          g_rgba=g_rgba, g_rgb=g_rgb, g_bg_rgb=g_bg, g_alpha=g_alpha, stream=_stream_ptr(dev))
            if ctx.deterministic:
                # bitwise-reproducible gradients from exact int64 sums (8 B of scratch per gradient element)
                nbytes = _lib.deterministic_scratch_bytes(d)
                scratch = torch.empty(nbytes, device=dev, dtype=torch.uint8)
                _lib.check(lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), scratch.data_ptr(), nbytes))
            else:
                _lib.check(lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)))
        return (g_rgba, g_rgb, g_alpha, g_bg) + (None,) * 11


def _mpi_ref(mpi) -> torch.Tensor:
    """The tensor of `mpi` = [rgba, rgb, alpha, bg_rgb] whose shape [M,N,_,Ht,Wt] and device a render takes: rgba, or the alpha of a
    factored MPI."""
    rgba, _, alpha, _ = mpi
    return alpha if rgba is None else rgba


def _mpi_desc(mpi, V, H, W, options, **fields):
    """Descriptor of a render of the MPI tensors `mpi` = [rgba, rgb, alpha, bg_rgb] (None where absent) from V views of H x W pixels:
    sizes, options and MPI pointers, plus the other descriptor `fields` (tensors or values, see _lib.make_desc)."""
    ref = _mpi_ref(mpi)
    return _lib.make_desc(options=options, M=ref.shape[0], V=V, N=ref.shape[1], Ht=ref.shape[-2], Wt=ref.shape[-1], H=H, W=W,
                          rgba=mpi[0], rgb=mpi[1], alpha=mpi[2], bg_rgb=mpi[3], **fields)


def _render_fwd(d, occ: Optional["Occupancy"], device):
    """Launch the forward `d` describes on `device`'s current stream; with an Occupancy `occ`, with empty-space skipping."""
    lib = _lib.load()
    with torch.cuda.device(device):
        d.stream = _stream_ptr(device)
        if occ is not None:
            _lib.check(lib.gmpi_mpi_render_fwd_skip_ex(ctypes.byref(d), occ.data_ptr(), occ.nbytes))
        else:
            _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)))


def _renders_natively(mpi, V, H, W, options, native):
    """Whether the MPI tensors `mpi` = [rgba, rgb, alpha, bg_rgb] (None where absent) render natively with the element-type option
    `native` (OPT_MPI_F16, OPT_MPI_U8): when they get the kernel plan a fresh fp32 allocation of their shape would get, so that the
    output is bitwise the render of their fp32 conversion."""
    fp32 = _mpi_desc(mpi, V, H, W, options)
    fp32.rgba = fp32.rgb = fp32.alpha = fp32.bg_rgb = None     # a fresh, aligned allocation
    return _lib.fwd_plan(fp32)[0] == _lib.fwd_plan(_mpi_desc(mpi, V, H, W, options | native))[0]


def _half_mpi(mpi, V, H, W, options):
    """The MPI tensors `mpi` = [rgba, rgb, alpha, bg_rgb] (None where absent) as contiguous fp16 when the call renders them natively
    (GMPI_MPI_F16), else None (the call upcasts them to fp32, as it always did).  Native when every MPI tensor is torch.float16,
    autograd does not record for them (the backward is fp32), and the fp16 MPI gets the kernel plan its fp32 upcast would get (the
    staged kernels need Wt % 8 == 0 and 16-byte aligned bases in fp16): the output is then bitwise the upcast's."""
    ts = [t for t in mpi if t is not None]
    if not all(t.dtype == torch.float16 for t in ts):
        return None
    if torch.is_grad_enabled() and any(t.requires_grad for t in ts):
        return None
    # detached: under no_grad an fp16 tensor may still carry requires_grad, and the native path has no backward
    half = [None if t is None else t.detach().contiguous() for t in mpi]
    return half if _renders_natively(half, V, H, W, options, _lib.OPT_MPI_F16) else None


_unorm8_tables = {}


def unorm8_to_float(x: torch.Tensor) -> torch.Tensor:
    """The fp32 MPI an 8-bit one stands for: code b -> b / 255 rounded to nearest, what the reference's mpi_from_plane_imgs computes
    (astype(np.float32) / 255.0, mpi_utils.py:336-337) and what GMPI_MPI_U8 renders.  A lookup in the 256-entry table of torch's CPU
    division, which rounds each quotient once; x.float() / 255 on a CUDA tensor multiplies by RN(1/255) instead, which differs in the
    last bit for 126 of the 256 codes."""
    t = _unorm8_tables.get(x.device)
    if t is None:
        t = _unorm8_tables[x.device] = (torch.arange(256, dtype=torch.float32) / 255).to(x.device)
    return t[x.int()]


def _check_unorm8(mpi):
    """unorm8=True takes an expanded torch.uint8 rgba: TypeError for anything else."""
    if mpi[0] is None or any(t is not None for t in mpi[1:]):
        raise TypeError("unorm8=True renders an expanded torch.uint8 rgba (code b = b / 255); got a factored MPI")
    if mpi[0].dtype != torch.uint8:
        raise TypeError(f"unorm8=True renders an expanded torch.uint8 rgba (code b = b / 255); got rgba of dtype {mpi[0].dtype}")


def _unorm8_mpi(mpi, V, H, W, options):
    """unorm8=True: the uint8 rgba of `mpi` = [rgba, rgb, alpha, bg_rgb] as the forward reads it, and its options.  Native (contiguous
    uint8 with GMPI_MPI_U8) when the uint8 MPI gets the kernel plan a fresh fp32 allocation of its shape would get (the staged kernels
    need Wt % 16 == 0 and a 16-byte aligned base in uint8), else its fp32 conversion (unorm8_to_float): the output is bitwise the
    render of that conversion either way."""
    _check_unorm8(mpi)
    u8 = [mpi[0].contiguous(), None, None, None]
    if _renders_natively(u8, V, H, W, options, _lib.OPT_MPI_U8):
        return u8, options | _lib.OPT_MPI_U8
    return [unorm8_to_float(u8[0]), None, None, None], options


def _launch_mpi(mpi, V, H, W, options, unorm8=False):
    """The MPI tensors `mpi` = [rgba, rgb, alpha, bg_rgb] (None where absent) as the forward reads them, and its options: with unorm8,
    see _unorm8_mpi; else contiguous fp16 with GMPI_MPI_F16 where _half_mpi renders them natively, else contiguous fp32."""
    if unorm8:
        return _unorm8_mpi(mpi, V, H, W, options)
    half = _half_mpi(mpi, V, H, W, options)
    if half is not None:
        return half, options | _lib.OPT_MPI_F16
    return [None if t is None else _as_f32c(t) for t in mpi], options


_warned_direct = set()


def _warn_if_direct(d):
    """Surface the direct-kernel performance cliff (several times slower than the TMA-staged kernels) of the forward descriptor `d`
    is about to launch, once per shape, MPI dtype and MPI base alignment."""
    key = (d.M, d.V, d.N, d.Ht, d.Wt, d.H, d.W, d.options & (_lib.OPT_MPI_F16 | _lib.OPT_MPI_U8)) + \
        tuple((p or 0) & 15 for p in (d.rgba, d.rgb, d.alpha, d.bg_rgb))
    if key in _warned_direct:
        return
    _warned_direct.add(key)
    plan, why = _lib.fwd_plan(d)
    if plan == _lib.PLAN_DIRECT and (why & ~2 or d.V * d.N * d.H * d.W >= 1 << 26):   # "few tiles" only matters when the problem is not tiny
        reasons = "; ".join(t for b, t in _lib.WHY.items() if why & b)
        warnings.warn(f"ml_gmpi_b200: rendering V={d.V} N={d.N} tex={d.Ht}x{d.Wt} img={d.H}x{d.W} with the direct (one thread per "
                      f"pixel) kernels, several times slower than the TMA-staged path: {reasons}", RuntimeWarning, stacklevel=4)


def _options(align_corners, check_last_plane, color_minus1_1, u8_round=False, early_stop=None):
    return (_lib.OPT_ALIGN_CORNERS if align_corners else 0) | (_lib.OPT_CHECK_LAST_PLANE if check_last_plane else 0) \
        | (_lib.OPT_COLOR_MINUS1_1 if color_minus1_1 else 0) | (_lib.OPT_U8_ROUND_HALF_UP if u8_round else 0) \
        | (_lib.OPT_EARLY_STOP if early_stop is not None else 0)


def _check_forward_only(option: str, is_set: bool, *inputs):
    """The backward needs every plane: early_stop drops the planes behind opaque content, and skip_empty the empty ones whose
    transmittance the training forward saves.  Refuse a set `option` where autograd would record."""
    if is_set and torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in inputs):
        why = " (it skips the planes the backward needs)" if option == "early_stop" else ""
        raise RuntimeError(f"ml_gmpi_b200: {option} is forward-only{why}; render under torch.no_grad() or from inputs that do not "
                           "require grad")


class Occupancy:
    """The occupancy map of one MPI stack (build_occupancy): one bit per 8 x 8 texel block of every (MPI, plane), set when a texel of
    the block is not empty (alpha not +0, or a colour value not finite; gmpi_mpi_build_occupancy).  It remembers the tensors it was
    built from (data pointer, shape, dtype and autograd version counter) and raises when a render hands it other tensors, or the
    same ones after an in-place change: a stale map would skip texels that are no longer empty."""

    def __init__(self, occ: torch.Tensor, nbytes: int, mpi):
        self.occ, self.nbytes = occ, nbytes
        self._stamp = self._stamp_of(mpi)

    @staticmethod
    def _stamp_of(mpi):
        return tuple(None if t is None else (t.data_ptr(), tuple(t.shape), t.dtype, t._version) for t in mpi)

    def data_ptr(self) -> int:
        return self.occ.data_ptr()

    def check(self, mpi):
        if self._stamp_of(mpi) != self._stamp:
            raise RuntimeError("ml_gmpi_b200: this Occupancy was built from other MPI tensors, or they were changed in place since; "
                               "build it again (build_occupancy)")


def build_occupancy(*, rgba=None, rgb=None, alpha=None, bg_rgb=None, flags: Optional[torch.Tensor] = None,
                    unorm8: bool = False) -> Occupancy:
    """The occupancy map of an expanded MPI rgba [M,N,4,Ht,Wt], or of a factored one (rgb [M,3,Ht,Wt], alpha [M,N,1,Ht,Wt], bg_rgb),
    fp32 or fp16, for render_views / render_views_factored / render_frames(skip_empty=...).  One streaming pass over the MPI (the
    factored MPI's colour is read once, its alpha per plane).  `flags` (expanded MPI): also OR in the range-check bits check_range
    sets, from the same pass.  unorm8=True: rgba is an 8-bit MPI (render_views(unorm8=True)); the pass reads its alpha bytes only,
    and every code is inside [0, 1], so there are no range bits to set."""
    mpi = [rgba, rgb, alpha, bg_rgb]
    ref = _mpi_ref(mpi)
    _require_cuda(ref)
    ts = [t for t in mpi if t is not None]
    if unorm8:
        _check_unorm8(mpi)
        launch, options = [rgba.detach().contiguous(), None, None, None], _lib.OPT_MPI_U8
    else:
        half = all(t.dtype == torch.float16 for t in ts)     # the map of an fp16 MPI is the map of its fp32 upcast
        launch = [None if t is None else (t.detach().contiguous() if half else _as_f32c(t.detach())) for t in mpi]
        options = _lib.OPT_MPI_F16 if half else 0
    d = _mpi_desc(launch, 1, 1, 1, options)
    n = _lib.occupancy_bytes(d)
    dev = ref.device
    occ = torch.empty((n + 3) // 4, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        d.flags = flags.data_ptr() if flags is not None else None
        d.stream = _stream_ptr(dev)
        _lib.check(_lib.load().gmpi_mpi_build_occupancy(ctypes.byref(d), occ.data_ptr(), n))
    return Occupancy(occ, n, mpi)


def _occupancy_for(skip_empty, mpi, unorm8=False) -> Optional[Occupancy]:
    """skip_empty of a render: False -> None; True -> a map built for this call; an Occupancy -> itself, if it describes `mpi`."""
    if skip_empty is False or skip_empty is None:
        return None
    if skip_empty is True:
        if unorm8:
            return build_occupancy(rgba=mpi[0], unorm8=True)
        return build_occupancy(rgba=mpi[0], rgb=mpi[1], alpha=mpi[2], bg_rgb=mpi[3])
    if not isinstance(skip_empty, Occupancy):
        raise TypeError(f"skip_empty must be a bool or an Occupancy, got {type(skip_empty).__name__}")
    skip_empty.check(mpi)
    return skip_empty


def render_views(rgba, dhw, view2mpi, ray_dir, eye, z_dir, *, align_corners=True, check_last_plane=False,
                 color_minus1_1=False, flags: Optional[torch.Tensor] = None, view_group: int = 1, early_stop: Optional[float] = None,
                 deterministic: Optional[bool] = None, skip_empty: Union[bool, Occupancy] = False, unorm8: bool = False):
    """Functional form on packed tensors (no list handling, no host sync).
    rgba [M,N,4,Ht,Wt], dhw [M,N,3], view2mpi [V] int32, ray_dir [V,3,H,W], eye/z_dir [V,3].
    Returns (color [V,3,H,W], depth [V,1,H,W]); `flags` (uint32 tensor of 1, int32 storage) is OR-ed into.
    view_group > 1: every view_group consecutive views share one MPI (tile-order hint: L2 reuse, see the C header).
    early_stop = tau in [0, 1): a pixel composites no further plane once its transmittance |T| <= tau (each colour channel moves by
    at most tau, 2 tau in [-1,1]; see gmpi_render_desc.early_stop).  Forward only: refused when an input requires grad.
    deterministic: the backward returns bitwise-reproducible gradients (exact int64 sums in a scratch of 8 B per gradient element,
    gmpi_mpi_render_bwd_deterministic_ex); None follows torch.are_deterministic_algorithms_enabled() at the time of this call.
    skip_empty: empty-space skipping (gmpi_mpi_render_fwd_skip_ex): the staged kernel does not load or composite the (tile, plane)
    boxes whose texels all have alpha +0 and finite colour; bitwise the same output.  True builds the map for this call
    (build_occupancy, one pass over the MPI); an Occupancy is reused.  Forward only: refused when an input requires grad.
    unorm8=True: rgba is an 8-bit MPI (torch.uint8, TypeError otherwise) whose code b stands for b / 255, the planar RGBA8 plane images
    of the reference's mpi_from_plane_imgs.  Rendered natively (GMPI_MPI_U8: a quarter of the fp32 bytes, no fp32 copy) where the
    kernel plan allows, else from its fp32 conversion; the output is bitwise render_views(unorm8_to_float(rgba)) either way.  With
    unorm8=False a uint8 rgba is upcast without scaling, as before."""
    return _render_views([rgba, None, None, None], dhw, view2mpi, ray_dir, eye, z_dir, align_corners, check_last_plane, color_minus1_1,
                         flags, view_group, early_stop, deterministic, skip_empty, unorm8)


def render_views_factored(rgb, alpha, dhw, view2mpi, ray_dir, eye, z_dir, *, bg_rgb=None, align_corners=True,
                          check_last_plane=False, color_minus1_1=False, flags: Optional[torch.Tensor] = None, view_group: int = 1,
                          early_stop: Optional[float] = None, deterministic: Optional[bool] = None,
                          skip_empty: Union[bool, Occupancy] = False):
    """The same render from the generator's FACTORED output (networks_cond_on_pos_enc.py:950-975,984): one colour image
    rgb [M,3,Ht,Wt] shared by all planes (bg_rgb [M,3,Ht,Wt]: the last plane's own colour under torgba_sep_background) and
    alpha [M,N,1,Ht,Wt] -- what the reference expands to [M,N,4,Ht,Wt] (and copies per view, train.py:553-558,733-738) before
    rendering.  Output identical to render_views on the expanded stack, 4x fewer HBM bytes; differentiable w.r.t. rgb, alpha
    and bg_rgb (d/d rgb is the sum over the planes that share it).  early_stop, deterministic, skip_empty: as in render_views."""
    return _render_views([None, rgb, alpha, bg_rgb], dhw, view2mpi, ray_dir, eye, z_dir, align_corners, check_last_plane, color_minus1_1,
                         flags, view_group, early_stop, deterministic, skip_empty)


def _check_factored_shapes(mpi):
    """The shapes of a factored MPI `mpi` = [None, rgb, alpha, bg_rgb] (an expanded one passes)."""
    rgba, rgb, alpha, bg_rgb = mpi
    if rgba is None:
        assert rgb.ndim == 4 and rgb.shape[1] == 3 and alpha.ndim == 5 and alpha.shape[2] == 1 and rgb.shape[0] == alpha.shape[0] \
            and rgb.shape[-2:] == alpha.shape[-2:], f"expected rgb [M,3,Ht,Wt] and alpha [M,N,1,Ht,Wt], got {rgb.shape}, {alpha.shape}"
        assert bg_rgb is None or bg_rgb.shape == rgb.shape, f"bg_rgb must have rgb's shape, got {bg_rgb.shape}"


def _render_views(mpi, dhw, view2mpi, ray_dir, eye, z_dir, align_corners, check_last_plane, color_minus1_1, flags, view_group,
                  early_stop, deterministic, skip_empty, unorm8=False):
    """render_views of the MPI tensors `mpi` = [rgba, rgb, alpha, bg_rgb] (None where absent), and render_views_factored."""
    _check_forward_only("early_stop", early_stop is not None, *mpi)
    _check_forward_only("skip_empty", skip_empty is not False and skip_empty is not None, *mpi)
    ref = _mpi_ref(mpi)
    _require_cuda(ref)
    _check_factored_shapes(mpi)
    if flags is None:
        flags = _zero_flags(ref.device)
    V, _, H, W = ray_dir.shape
    if unorm8:
        _check_unorm8(mpi)
    occ = _occupancy_for(skip_empty, mpi, unorm8)
    mpi, options = _launch_mpi(mpi, V, H, W, _options(align_corners, check_last_plane, color_minus1_1, early_stop=early_stop), unorm8)
    _warn_if_direct(_mpi_desc(mpi, V, H, W, options))
    return _RenderFn.apply(*mpi, _as_f32c(dhw), view2mpi, _as_f32c(ray_dir), _as_f32c(eye), _as_f32c(z_dir),
                           options, flags, int(view_group), early_stop, deterministic, occ)


class TrainPlan(NamedTuple):
    """The kernels of a training render (train_plan): for each pass _lib.PLAN_STAGED (the TMA-staged forward, the box backward) or
    _lib.PLAN_DIRECT (the direct kernels: one thread per pixel forward, two passes over every plane backward), the GMPI_WHY_* bits of
    every reason it is not the staged kernel, and those reasons in words (_lib.WHY)."""
    forward: int
    forward_why: int
    forward_reasons: Tuple[str, ...]
    backward: int
    backward_why: int
    backward_reasons: Tuple[str, ...]


# What a descriptor holds for a buffer the render allocates itself (torch.empty / empty_like: a fresh allocation, 512-byte aligned):
# the plan queries read its alignment, never its memory.
_FRESH_BUFFER = 512


def train_plan(*, dhw, view2mpi, ray_dir, eye, z_dir, rgba=None, rgb=None, alpha=None, bg_rgb=None, align_corners=True,
               check_last_plane=False, color_minus1_1=False, view_group: int = 1, deterministic: Optional[bool] = None) -> TrainPlan:
    """Which kernels the training render of these inputs gets, asked before it runs: render_views(rgba, ...) or
    render_views_factored(rgb, alpha, ..., bg_rgb=...) with the same tensors and keywords, with autograd recording for the MPI, then
    its backward (gmpi_mpi_render_fwd_plan_ex and gmpi_mpi_render_bwd_plan_ex).  The descriptor is the one the render launches: the
    MPI tensors as _launch_mpi hands them to the kernels (a copy where they are not contiguous fp32), and the transmittance and
    gradient buffers the render allocates, which are fresh and aligned.  The MPI tensors need not be on the GPU and nothing is
    launched; no other input is read.  deterministic (None: torch.are_deterministic_algorithms_enabled()): the deterministic backward
    makes the same kernel choice, and its scratch-size query must accept the call too.  Raises ValueError when no MPI tensor requires
    grad (the render then has no backward), and GmpiLibraryError where the backward call would refuse the inputs."""
    mpi = [rgba, rgb, alpha, bg_rgb]
    _check_factored_shapes(mpi)
    if not any(t is not None and t.requires_grad for t in mpi):
        raise ValueError("train_plan answers for a training render: no MPI tensor requires grad, so the render has no backward")
    V, _, H, W = ray_dir.shape
    with torch.enable_grad():            # what the training render sees: autograd records for the MPI
        mpi, options = _launch_mpi(mpi, V, H, W, _options(align_corners, check_last_plane, color_minus1_1))
    fresh = lambda t: None if t is None else _FRESH_BUFFER
    d = _mpi_desc(mpi, V, H, W, options, view_group=int(view_group), transmittance=_FRESH_BUFFER)
    fwd, fwd_why = _lib.fwd_plan(d)
    # _RenderFn.backward: the same descriptor with GMPI_ZERO_GRAD and an empty_like gradient of every MPI tensor
    d.options |= _lib.OPT_ZERO_GRAD
    d.g_rgba, d.g_rgb, d.g_alpha, d.g_bg_rgb = (fresh(t) for t in mpi)
    bwd, bwd_why = _lib.bwd_plan(d)
    if torch.are_deterministic_algorithms_enabled() if deterministic is None else deterministic:
        _lib.deterministic_scratch_bytes(d)
    return TrainPlan(fwd, fwd_why, tuple(_lib.reasons(fwd_why)), bwd, bwd_why, tuple(_lib.reasons(bwd_why)))


def expand_factored(rgb, alpha, bg_rgb=None):
    """[M,3,Ht,Wt] + [M,N,1,Ht,Wt] -> [M,N,4,Ht,Wt], the generator's expand + cat (networks_cond_on_pos_enc.py:950-975):
    what the reference renders from; here only tests and callers that need the expanded stack use it."""
    N = alpha.shape[1]
    col = rgb.unsqueeze(1).expand(-1, N, -1, -1, -1)
    if bg_rgb is not None:
        col = torch.cat([col[:, : N - 1], bg_rgb.unsqueeze(1)], dim=1)
    return torch.cat([col, alpha], dim=2).contiguous()


def render_frames(*, dhw, view2mpi, rgba=None, rgb=None, alpha=None, bg_rgb=None, ray_dir=None, eye=None, z_dir=None, cam=None,
                  align_corners=True, check_last_plane=False, video: Optional[dict] = None, u8_round=False,
                  flags: Optional[torch.Tensor] = None, view_group: int = 1, H: Optional[int] = None, W: Optional[int] = None,
                  early_stop: Optional[float] = None, skip_empty: Union[bool, Occupancy] = False, unorm8: bool = False):
    """Inference-only render with the opt-in fast paths of the C ABI (no autograd):
      unorm8=True    rgba is an 8-bit MPI, code b = b / 255 (see render_views).
      skip_empty=True or an Occupancy   empty-space skipping, bitwise the same frames (see render_views).
      cam [V,16]     rays generated in the kernel from the pinhole camera (see camera.cam_params) instead of ray_dir/eye/z_dir;
      video={"near": ray_start, "far": ray_end, "depth": True}   uint8 HWC frames as render_video.py:118-126 builds them:
                     returns (rgb_u8 [V,H,W,3], depth_u8 [V,H,W,1] or None); otherwise (color in [-1,1], depth) fp32.
      early_stop=tau in [0, 1)   early ray termination: a pixel composites no further plane once its transmittance |T| <= tau
                     (colour in [-1,1] moves by at most 2 tau per channel, a uint8 code by at most one; see render_views).
    """
    mpi = [rgba, rgb, alpha, bg_rgb]
    ref = _mpi_ref(mpi)
    _require_cuda(ref)
    _lib.load()                     # a missing library is reported before the arguments are checked
    dev = ref.device
    if cam is not None:
        V = cam.shape[0]
        assert H is not None and W is not None, "pass H and W with cam"
        cam = _as_f32c(cam)
    else:
        V, _, H, W = ray_dir.shape
        ray_dir, eye, z_dir = _as_f32c(ray_dir), _as_f32c(eye), _as_f32c(z_dir)
    if flags is None:
        flags = _zero_flags(dev)
    color = depth = v_rgb = v_depth = None
    near = rng = 0.0
    if video is not None:
        v_rgb = torch.empty((V, H, W, 3), device=dev, dtype=torch.uint8)
        if video.get("depth", True):
            v_depth = torch.empty((V, H, W, 1), device=dev, dtype=torch.uint8)
        near = float(np.float32(video["near"]))
        rng = float(np.float32(video["far"] - video["near"]))            # the python-double difference, rounded once (numpy weak scalar)
    else:
        color = torch.empty((V, 3, H, W), device=dev, dtype=torch.float32)
        depth = torch.empty((V, 1, H, W), device=dev, dtype=torch.float32)
    if unorm8:
        _check_unorm8(mpi)
    occ = _occupancy_for(skip_empty, mpi, unorm8)
    mpi, options = _launch_mpi(mpi, V, H, W, _options(align_corners, check_last_plane, True, u8_round, early_stop), unorm8)
    _render_fwd(_mpi_desc(mpi, V, H, W, options, view_group=int(view_group), depth_near=near, depth_range=rng, view2mpi=view2mpi,
                          dhw=_as_f32c(dhw), ray_dir=ray_dir, eye=eye, z_dir=z_dir, cam=cam, color=color, depth=depth, video_rgb=v_rgb,
                          video_depth=v_depth, flags=flags, early_stop=early_stop), occ, dev)
    return (v_rgb, v_depth) if video is not None else (color, depth)


def check_range(rgba: torch.Tensor, flags: torch.Tensor) -> None:
    """One streaming pass: RGBA/alpha in [0,1] (mpi_renderer.py:447-449, mpi.py:185-187) -> flag bits.  rgba is contiguous fp32, or
    contiguous fp16 (the flags of the fp32 check on its upcast)."""
    lib = _lib.load()
    M, N, _, Ht, Wt = rgba.shape
    check = lib.gmpi_mpi_check_range_f16 if rgba.dtype == torch.float16 else lib.gmpi_mpi_check_range
    with torch.cuda.device(rgba.device):
        _lib.check(check(rgba.data_ptr(), M, N, Ht, Wt, flags.data_ptr(), _stream_ptr(rgba.device)))


class MPI(nn.Module):
    """`validate`:
         "full"  (default) every data-dependent assert of the reference is evaluated on the device
                 (alpha range scan, plane-behind-camera, rays leaving the last plane) and raised
                 after ONE host sync per call (the reference syncs six or more times);
         "defer" the geometric flags are still computed inside the render kernel (free) but nothing
                 is scanned or synced; read them later with `.raise_if_flagged()`;
         "off"   like "defer" without the last-plane check.
    `deterministic`: bitwise-reproducible gradients w.r.t. batch_rgba (see render_views); None (default) follows
    torch.use_deterministic_algorithms at each forward.
    `skip_empty`: empty-space skipping (render_views(skip_empty=...)), forward only: refused when batch_rgba requires grad under
    autograd.  With validate="full" the occupancy map comes from the range check's pass; the flags and messages are unchanged.
    """

    def __init__(self, align_corners=True, validate: str = "full", deterministic: Optional[bool] = None, skip_empty: bool = False):
        super().__init__()
        assert validate in ("full", "defer", "off"), validate
        self._align_corners = align_corners
        self.validate = validate
        self.deterministic = deterministic
        self.skip_empty = bool(skip_empty)
        self._flags = None
        self._flag_ctx = None

    # -- reference: MPI.check_shapes, mpi.py:161-216 (shape part; the alpha range is checked on the device)
    def check_shapes(self, *, batch_rgba, batch_dhw, batch_ray_dir, batch_eye_pos, batch_z_dir, separate_background):
        assert (batch_rgba.ndim == 5) and (batch_rgba.shape[2] == 4), (
            f"Expected rgba to be of shape (#mpi, #planes, 4, texture_height, texture_width), "
            f"but instead got {batch_rgba.shape}")
        assert ((batch_dhw.ndim == 3) and (batch_dhw.shape[0] == batch_rgba.shape[0])
                and (batch_dhw.shape[1] == batch_rgba.shape[1]) and (batch_dhw.shape[2] == 3)), (
            f"Expected dhw to be of shape (#mpi, #planes, 3), but instead got {batch_dhw.shape} (rgba: {batch_rgba.shape})")
        assert len(batch_ray_dir) == batch_rgba.shape[0], f"{len(batch_ray_dir)}, {batch_rgba.shape[0]}"
        assert len(batch_eye_pos) == batch_rgba.shape[0], f"{len(batch_eye_pos)}, {batch_rgba.shape[0]}"
        assert len(batch_z_dir) == batch_rgba.shape[0], f"{len(batch_z_dir)}, {batch_rgba.shape[0]}"
        for i in range(len(batch_ray_dir)):
            assert (batch_ray_dir[i].ndim == 4) and (batch_ray_dir[i].shape[1] == 3), (
                f"Expected ray_dir to be of shape (minibatch, 3, image_height, image_width), "
                f"but instead got {batch_ray_dir[i].shape} for {i} th elem.")
            assert (batch_eye_pos[i].ndim == 2) and (batch_eye_pos[i].shape[1] == 3), (
                f"Expected eye_pos to be of shape (minibatch, 3), but instead got {batch_eye_pos[i].shape} for {i} th elem.")
            assert (batch_z_dir[i].ndim == 2) and (batch_z_dir[i].shape[1] == 3), (
                f"Expected z_dir to be of shape (minibatch, 3), but instead got {batch_z_dir[i].shape} for {i} th elem.")
        if separate_background is not None:
            assert separate_background.ndim == 4 and separate_background.shape[1] == 3, (
                f"Expect background to be of shape (#mpi, 3, h, w), but instead get {separate_background.shape}.")

    @staticmethod
    def pack_views(batch_ray_dir, batch_eye_pos, batch_z_dir, device):
        """mpi.py:334-354 without the copies of the MPI: views stay MPI-major and a [V] int32 index
        replaces expand+cat of rgba/dhw."""
        counts = [int(r.shape[0]) for r in batch_ray_dir]
        if all(c == 1 for c in counts):
            view2mpi = torch.arange(len(counts), dtype=torch.int32, device=device)
        else:
            view2mpi = torch.repeat_interleave(torch.arange(len(counts), dtype=torch.int32),
                                               torch.tensor(counts)).to(device=device, dtype=torch.int32)
        cat = (lambda xs: xs[0] if len(xs) == 1 else torch.cat(xs, dim=0))
        return view2mpi, cat(list(batch_ray_dir)), cat(list(batch_eye_pos)), cat(list(batch_z_dir))

    @staticmethod
    def view_group_of(batch_ray_dir) -> int:
        """k when every MPI is rendered from the same number k > 1 of views (the expand of train.py:733-738 /
        train_helpers.py:181-186, a video sweep of one MPI): the kernels then order tiles for L2 reuse.  Else 1."""
        counts = {int(r.shape[0]) for r in batch_ray_dir}
        k = counts.pop() if len(counts) == 1 else 1
        return k if k > 1 else 1

    def forward(self, *, batch_rgba: torch.Tensor, batch_dhw: torch.Tensor, batch_ray_dir: List[torch.Tensor],
                batch_eye_pos: List[torch.Tensor], batch_z_dir: List[torch.Tensor],
                separate_background: Union[None, torch.Tensor], assert_not_out_of_last_plane: bool = False,
                c2w_mat: torch.Tensor = None, sphere_c: np.ndarray = None):
        self.check_shapes(batch_rgba=batch_rgba, batch_dhw=batch_dhw, batch_ray_dir=batch_ray_dir,
                          batch_eye_pos=batch_eye_pos, batch_z_dir=batch_z_dir, separate_background=separate_background)
        _require_cuda(batch_rgba, "ml_gmpi_b200.MPI renders")
        dev = batch_rgba.device
        view2mpi, ray_dir, eye, z_dir = self.pack_views(batch_ray_dir, batch_eye_pos, batch_z_dir, dev)
        # an fp16 MPI stays fp16: render_views renders it natively where it can (and upcasts it where it cannot)
        rgba = batch_rgba.contiguous() if batch_rgba.dtype == torch.float16 else _as_f32c(batch_rgba)
        flags = _zero_flags(dev)
        occ = False
        if self.skip_empty:
            _check_forward_only("skip_empty", True, batch_rgba)
            occ = build_occupancy(rgba=rgba, flags=flags if self.validate == "full" else None)
        elif self.validate == "full":
            check_range(rgba.detach(), flags)
        color, depth = render_views(rgba, batch_dhw.to(dev), view2mpi, ray_dir.to(dev), eye.to(dev), z_dir.to(dev),
                                    align_corners=self._align_corners,
                                    check_last_plane=bool(assert_not_out_of_last_plane) and self.validate != "off",
                                    flags=flags, view_group=self.view_group_of(batch_ray_dir), deterministic=self.deterministic,
                                    skip_empty=occ)
        self._flags = flags
        self._flag_ctx = (batch_dhw, eye, c2w_mat, sphere_c)
        if self.validate == "full":
            self.raise_if_flagged(ignore=_lib.FLAG_RGBA_RANGE)   # rgba range is MPIRenderer.render's assert
        return color, depth

    def last_flags(self) -> int:
        """Flag word of the most recent forward (one host sync)."""
        return 0 if self._flags is None else int(self._flags.item()) & 0xFFFFFFFF

    def raise_if_flagged(self, ignore: int = 0):
        f = self.last_flags() & ~ignore
        if f == 0:
            return
        dhw, eye, c2w, sphere_c = self._flag_ctx
        if f & _lib.FLAG_ALPHA_RANGE:
            raise AssertionError("Expected alpha to be within the the range [0, 1]")             # mpi.py:185-187
        if f & _lib.FLAG_RGBA_RANGE:
            raise AssertionError("MPI rgba outside [0, 1]")                                       # mpi_renderer.py:447-449
        if f & _lib.FLAG_PLANE_BEHIND_EYE:
            raise AssertionError(f"Camera must be placed closer to origin than MPI. {dhw[..., 0]}, {eye[0, ...]}")  # mpi.py:70-72
        if f & _lib.FLAG_LAST_PLANE_OOB:
            msg = f"Ray's U/V direction goes out of plane at {dhw[:, -1, 0]}"                    # mpi.py:106-109
            if c2w is not None and sphere_c is not None:
                msg += f"; c2w: {c2w.detach().cpu().numpy().tolist()}"
            raise MPIOutOfPlaneError(msg)
