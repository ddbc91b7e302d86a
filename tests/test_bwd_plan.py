"""The backward plan: which kernel a training call's backward takes (the staged box kernel or the two-pass direct kernel) and every
reason it does not take the box kernel, asked before the forward runs (gmpi_mpi_render_bwd_plan_ex, ml_gmpi_b200.train_plan).

One host function decides it for the launches of gmpi_mpi_render_bwd_ex and gmpi_mpi_render_bwd_deterministic_ex and for the query.
These CPU tests check each GMPI_WHY_* bit on fake pointers (the query reads their values only), that the bits combine and that the
box is exactly "forward plan staged and no backward reason", that the query refuses what the backward call refuses with the same code
and message, and that train_plan answers for the descriptor the render launches.  tests/test_gpu_bwd_plan.py checks on the GPU that
each backward launches the kernel its plan predicts."""
import ctypes
import itertools

import pytest
import torch

import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib
from testlib import forced_kernel, lib

TEX_WIDTH, FEW_TILES, MANY_PLANES, ALIGNMENT, FORCED = 1, 2, 4, 8, 16
NO_TRANSMITTANCE, IMG_WIDTH, GRAD_ALIGNMENT, MANY_PIXEL_PLANES = 32, 64, 128, 256
F16, U8, ES = _lib.OPT_MPI_F16, _lib.OPT_MPI_U8, _lib.OPT_EARLY_STOP
# the benchmark's shape, trained: an expanded MPI, its gradient and the saved transmittance at aligned fake addresses -> the box
SIZES = dict(M=4, V=4, N=96, Ht=1024, Wt=1024, H=1024, W=1024)
TRAIN = dict(rgba=16, g_rgba=32, transmittance=48)
# a factored MPI with a background plane, and its gradients
FACTORED = dict(rgba=None, g_rgba=None, rgb=64, alpha=80, bg_rgb=96, g_rgb=112, g_alpha=128, g_bg_rgb=144)


def _desc(**kw):
    return _lib.make_desc(**{**SIZES, **TRAIN, **kw})


def _plan(d):
    """(return value, why) of gmpi_mpi_render_bwd_plan_ex; why is 0xffffffff where the query does not write it."""
    why = ctypes.c_uint32(0xffffffff)
    return _lib.load().gmpi_mpi_render_bwd_plan_ex(ctypes.byref(d), ctypes.byref(why)), why.value


def _why(**kw):
    plan, why = _lib.bwd_plan(_desc(**kw))
    assert plan == (_lib.PLAN_STAGED if why == 0 else _lib.PLAN_DIRECT), (plan, why)
    return why


def test_each_backward_reason_sets_its_bit(lib):
    assert _why() == 0 and _why(**FACTORED) == 0 and _why(**dict(FACTORED, bg_rgb=None, g_bg_rgb=None)) == 0
    assert _why(transmittance=None) == NO_TRANSMITTANCE
    assert _why(W=68) == 0 and _why(W=66) == IMG_WIDTH and _why(W=1022) == IMG_WIDTH
    for ptrs in (dict(g_rgba=40), dict(transmittance=56), dict(FACTORED, g_rgb=120), dict(FACTORED, g_alpha=136),
                 dict(FACTORED, g_bg_rgb=152), dict(FACTORED, transmittance=8)):
        assert _why(**ptrs) == GRAD_ALIGNMENT, ptrs
    # NULL gradients count as aligned; only the gradients of the MPI's form are read
    assert _why(g_rgba=None) == 0 and _why(**dict(FACTORED, g_rgb=None, g_alpha=None, g_bg_rgb=None)) == 0
    assert _why(g_alpha=8) == 0 and _why(**dict(FACTORED, g_rgba=8)) == 0


def test_the_pixel_planes_of_the_transmittance(lib):
    """V*N = 2^31 - N takes the box; at 2^31 the backward takes the direct kernel, which refuses more than 65535 views: the query
    returns that refusal and still writes why."""
    assert _why(N=512, V=(1 << 22) - 1) == 0
    rc, why = _plan(_desc(N=512, V=1 << 22))
    assert rc == -3 and why == MANY_PIXEL_PLANES and b"65535" in _lib.load().gmpi_last_error()


def test_each_forward_reason_carries_through(lib):
    for kw, bit in ((dict(Wt=1022), TEX_WIDTH), (dict(V=1, H=270, W=768), FEW_TILES), (dict(N=513), MANY_PLANES),
                    (dict(rgba=8), ALIGNMENT), (dict(FACTORED, alpha=88), ALIGNMENT)):
        assert _why(**kw) == bit and _lib.fwd_plan(_desc(**kw))[1] == bit, kw
    with forced_kernel("direct"):
        assert _why() == FORCED
    with forced_kernel("staged"):
        assert _why(V=1, H=48, W=48) == 0


def test_reasons_combine(lib):
    assert _why(transmittance=None, W=66, g_rgba=40) == NO_TRANSMITTANCE | IMG_WIDTH | GRAD_ALIGNMENT
    assert _why(Wt=1022, rgba=8, transmittance=24, V=1, H=48, W=50) == TEX_WIDTH | ALIGNMENT | FEW_TILES | GRAD_ALIGNMENT | IMG_WIDTH
    with forced_kernel("direct"):
        assert _why(transmittance=None, N=600) == FORCED | NO_TRANSMITTANCE | MANY_PLANES


def test_box_exactly_when_the_forward_is_staged_and_no_backward_reason_holds(lib):
    for variant in ("auto", "direct", "staged"):
        with forced_kernel(variant):
            for V, N, Wt, H, W, rgba, trans, g_rgba in itertools.product((1, 4), (16, 512, 513), (1020, 1022, 1024), (48, 300, 1024),
                                                                         (1024, 1026), (None, 8, 16), (None, 16, 24), (None, 16, 40)):
                d = _lib.make_desc(M=2, V=V, N=N, Ht=1024, Wt=Wt, H=H, W=W, rgba=rgba, transmittance=trans, g_rgba=g_rgba)
                fwd_plan, fwd_why = _lib.fwd_plan(d)
                own = (NO_TRANSMITTANCE if trans is None else 0) | (IMG_WIDTH if W % 4 else 0) | \
                    (GRAD_ALIGNMENT if (trans or 0) % 16 or (g_rgba or 0) % 16 else 0)
                plan, why = _lib.bwd_plan(d)
                case = (variant, V, N, Wt, H, W, rgba, trans, g_rgba)
                assert why == fwd_why | own, case
                assert (plan == _lib.PLAN_STAGED) == (fwd_plan == _lib.PLAN_STAGED and own == 0), case


# ------------------------------------------------------------------------------------------------------------------------------
# refusals: the query refuses what gmpi_mpi_render_bwd_ex refuses before it launches, with the same code and message
# ------------------------------------------------------------------------------------------------------------------------------
GEOMETRY = dict(view2mpi=256, dhw=272, ray_dir=288, eye=304, z_dir=320, g_color=336)
REFUSED = {                     # name: (descriptor fields on top of SIZES, TRAIN and GEOMETRY, GMPI_ERR_* code)
    "F16": (dict(options=F16), 3), "U8": (dict(options=U8), 3), "ES": (dict(options=ES, early_stop=0.5), 3),
    "F16|U8": (dict(options=F16 | U8), 1), "F16 factored": (dict(FACTORED, options=F16), 3),
    "ES without transmittance": (dict(options=ES, early_stop=0.5, transmittance=None), 3),
    "cam": (dict(cam=352, ray_dir=None, eye=None, z_dir=None), 3),
    "N=0": (dict(N=0), 1), "W=0": (dict(W=0), 1), "V=-1": (dict(V=-1), 1), "M=0": (dict(M=0), 1),
    "texture of 2^31 texels": (dict(Ht=1 << 16, Wt=1 << 15), 3),
    "view_group=3": (dict(view_group=3), 1), "view_group=-1": (dict(view_group=-1), 1),
    # the direct kernel's limits, where it takes the direct kernel
    "65536 views": (dict(V=65536, H=64, W=64, transmittance=None), 3),
    "65536 views, factored": (dict(FACTORED, V=65536, H=64, W=66), 3),
    "image too tall": (dict(V=1, H=262141, W=4, N=8, transmittance=None), 3),
    "N beyond the stash": (dict(N=1500, H=64, W=64), 3),
}


@pytest.mark.parametrize("name", list(REFUSED))
def test_refusals_match_the_backward_call(name, lib):
    fields, code = REFUSED[name]
    d = _lib.make_desc(**{**SIZES, **TRAIN, **GEOMETRY, **fields})
    rc, why = _plan(d)
    plan_msg = lib.gmpi_last_error()
    assert rc == -code, (rc, plan_msg)
    assert plan_msg, name
    if d.V > 0 and torch.cuda.is_available():
        return      # the backward calls would launch a kernel on these host addresses if they accepted the descriptor
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == code and lib.gmpi_last_error() == plan_msg
    scratch = 1 << 12       # an aligned stand-in: a call that refuses reads none of it
    assert lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), scratch, 1 << 50) == code and lib.gmpi_last_error() == plan_msg


def test_the_query_asks_for_no_pointer(lib):
    """The backward call refuses a descriptor without rays or upstream gradient; the query answers for sizes, options and the
    pointers it reads."""
    assert _lib.bwd_plan(_lib.make_desc(**SIZES, transmittance=16)) == (_lib.PLAN_STAGED, 0)
    assert _lib.bwd_plan(_lib.make_desc(**SIZES)) == (_lib.PLAN_DIRECT, NO_TRANSMITTANCE)
    d = _lib.make_desc(**dict(SIZES, V=0))
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == 1 and _lib.bwd_plan(d) == (_lib.PLAN_DIRECT, NO_TRANSMITTANCE | FEW_TILES)
    rc, why = _plan(_lib.make_desc(**dict(SIZES, N=1500, V=0)))     # V = 0 launches nothing: no direct-kernel limit applies
    assert rc == _lib.PLAN_DIRECT and why == NO_TRANSMITTANCE | MANY_PLANES | FEW_TILES
    d.struct_bytes = 8
    assert _plan(d) == (-1, 0xffffffff) and b"struct_bytes" in lib.gmpi_last_error()
    assert lib.gmpi_mpi_render_bwd_plan_ex(None, None) == -1


# ------------------------------------------------------------------------------------------------------------------------------
# train_plan: the plans of the descriptor the render launches
# ------------------------------------------------------------------------------------------------------------------------------
def _inputs(form, tex=64, Wt=None, N=8, views=4, img=256, W=None, grad=True, misalign=None, dtype=torch.float32):
    """CPU tensors of a training render of two MPIs: the MPI of `form`, requiring grad, and the geometry of `views` views."""
    gen = torch.Generator().manual_seed(3)
    hw = (tex, Wt or tex)

    def rand(*shape, name):
        t = torch.rand(shape, generator=gen).to(dtype)
        if name == misalign:            # 8 bytes past a 16-byte boundary
            buf = torch.empty(t.numel() + 4, dtype=dtype)
            start = (8 - buf.data_ptr() % 16) % 16 // buf.element_size()
            t = buf[start:start + t.numel()].view(shape).copy_(t)
            assert t.data_ptr() % 16 == 8
        return t.requires_grad_(grad)

    if form == "expanded":
        m = dict(rgba=rand(2, N, 4, *hw, name="rgba"))
    else:
        m = dict(rgb=rand(2, 3, *hw, name="rgb"), alpha=rand(2, N, 1, *hw, name="alpha"),
                 bg_rgb=rand(2, 3, *hw, name="bg_rgb") if form == "factored_bg" else None)
    geo = dict(dhw=torch.rand(2, N, 3), view2mpi=torch.arange(views, dtype=torch.int32) % 2, ray_dir=torch.rand(views, 3, img, W or img),
               eye=torch.rand(views, 3), z_dir=torch.rand(views, 3))
    return m, geo


def _c_desc(m, geo, options):
    """The descriptor of the training render built by hand: the MPI tensors as they are, gradients and transmittance at aligned
    addresses."""
    ref = m.get("rgba") if m.get("rgba") is not None else m["alpha"]
    V, _, H, W = geo["ray_dir"].shape
    grads = {"g_" + k: 1024 for k, t in m.items() if t is not None}
    return _lib.make_desc(options=options | _lib.OPT_ZERO_GRAD, M=ref.shape[0], V=V, N=ref.shape[1], Ht=ref.shape[-2], Wt=ref.shape[-1],
                          H=H, W=W, transmittance=2048, **m, **grads)


TRAIN_CASES = {"staged": {}, "W=66": dict(W=66, img=512),"few tiles": dict(views=1), "Wt=66": dict(Wt=66), "N=513": dict(N=513, tex=8)}


@pytest.mark.parametrize("deterministic", [None, False, True])
@pytest.mark.parametrize("case", list(TRAIN_CASES))
@pytest.mark.parametrize("form", ["expanded", "factored", "factored_bg"])
def test_train_plan_agrees_with_the_c_queries(form, case, deterministic, lib):
    m, geo = _inputs(form, **TRAIN_CASES[case])
    p = g.train_plan(**m, **geo, align_corners=True, deterministic=deterministic)
    d = _c_desc(m, geo, _lib.OPT_ALIGN_CORNERS)
    assert (p.forward, p.forward_why) == _lib.fwd_plan(d) and (p.backward, p.backward_why) == _lib.bwd_plan(d), p
    assert p.forward_reasons == tuple(_lib.WHY[b] for b in _lib.WHY if p.forward_why & b)
    assert p.backward_reasons == tuple(_lib.WHY[b] for b in _lib.WHY if p.backward_why & b)
    expect = {"staged": 0, "W=66": IMG_WIDTH, "few tiles": FEW_TILES, "Wt=66": TEX_WIDTH, "N=513": MANY_PLANES}[case]
    assert p.backward_why == expect and p.forward_why == expect & ~IMG_WIDTH, p


@pytest.mark.parametrize("form,tensor", [("expanded", "rgba"), ("factored", "alpha"), ("factored_bg", "bg_rgb")])
def test_train_plan_sees_the_tensors_the_render_launches(form, tensor, lib):
    """A misaligned fp32 MPI tensor is launched as it is: both passes take the direct kernels.  An fp64 one is launched from a fresh
    fp32 copy, whose alignment is the allocator's."""
    m, geo = _inputs(form, misalign=tensor)
    p = g.train_plan(**m, **geo)
    assert (p.forward_why, p.backward_why) == (ALIGNMENT, ALIGNMENT), p
    assert p.backward_reasons == ("an MPI base pointer is not 16-byte aligned",)
    m, geo = _inputs(form, misalign=tensor, dtype=torch.float64)
    assert g.train_plan(**m, **geo) == (_lib.PLAN_STAGED, 0, (), _lib.PLAN_STAGED, 0, ())


def test_train_plan_refuses_what_the_render_refuses(lib):
    m, geo = _inputs("expanded", grad=False)
    with pytest.raises(ValueError, match="no MPI tensor requires grad"):
        g.train_plan(**m, **geo)
    m, geo = _inputs("expanded", views=3)
    with pytest.raises(_lib.GmpiLibraryError, match="view_group=2 does not divide V=3"):
        g.train_plan(**m, **geo, view_group=2)
    m, geo = _inputs("factored", N=1500, tex=8)       # the direct backward's stash holds fewer planes
    with pytest.raises(_lib.GmpiLibraryError, match="exceed the backward stash"):
        g.train_plan(**m, **geo)
