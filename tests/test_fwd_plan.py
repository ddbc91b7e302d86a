"""The forward plan: which kernels a render takes (TMA-staged or direct) and every reason it does not take the staged ones.

One host function decides it for the launch and for every query (gmpi_mpi_render_fwd_plan, _plan_ex, _variant, and the Python
warning).  The CPU tests check each GMPI_WHY_* bit on null or fake pointers, that the three queries agree, and that the warning
sees every MPI tensor as it is launched.  The GPU test (pytest -m gpu) checks that each launch takes the kernel its query predicts,
observed through the early-stop statistics: at tau = 0 the staged kernel counts every (tile, plane) stage it walks, the direct
kernel none, and the colour is bitwise the same launch's without early stop."""
import ctypes
import itertools
import warnings

import pytest
import torch

from ml_gmpi_b200 import _lib, mpi, synth
from testlib import assert_bitwise, early_stop_stats, forced_kernel, lib, misaligned

TEX_WIDTH, FEW_TILES, MANY_PLANES, ALIGNMENT, FORCED = 1, 2, 4, 8, 16
F16 = _lib.OPT_MPI_F16
SIZES = dict(M=4, V=4, N=96, Ht=1024, Wt=1024, H=1024, W=1024)     # the benchmark's shape: staged


def _why(**kw):
    plan, why = _lib.fwd_plan(_lib.make_desc(**{**SIZES, **kw}))
    assert plan == (_lib.PLAN_STAGED if why == 0 else _lib.PLAN_DIRECT), (plan, why)
    return why


def test_each_reason_sets_its_bit(lib):
    assert _why() == 0
    assert _why(Wt=1022) == TEX_WIDTH
    assert _why(Wt=1020) == 0 and _why(Wt=1020, options=F16) == TEX_WIDTH and _why(Wt=1016, options=F16) == 0
    assert _why(V=1, H=300, W=768) == 0 and _why(V=1, H=270, W=768) == FEW_TILES      # 12 x 10 and 12 x 9 tiles of 64x30
    assert _why(N=512) == 0 and _why(N=513) == MANY_PLANES
    assert _why(M=(1 << 22) - 1, N=512) == 0 and _why(M=1 << 22, N=512) == MANY_PLANES    # M*N = 2^31 - 512, 2^31
    assert _why(M=1 << 30, N=2) == MANY_PLANES
    for ptrs in (dict(rgba=8), dict(rgb=8, alpha=16), dict(rgb=16, alpha=8), dict(rgb=16, alpha=32, bg_rgb=40)):
        assert _why(**ptrs) == ALIGNMENT, ptrs
        assert _why(**ptrs, options=F16) == ALIGNMENT, ptrs
    assert _why(rgba=16) == 0 and _why(rgb=16, alpha=32) == 0 and _why(rgb=16, alpha=32, bg_rgb=48) == 0
    assert _why(V=1, H=48, W=48, N=600, Wt=1022, rgba=8) == TEX_WIDTH | FEW_TILES | MANY_PLANES | ALIGNMENT


def test_forced_variants(lib):
    with forced_kernel("direct"):
        assert _why() == FORCED and _why(V=1, H=48, W=48) == FORCED | FEW_TILES
    with forced_kernel("staged"):
        assert _why(V=1, H=48, W=48) == 0 and _why(V=1, H=48, W=48, Wt=1022) == TEX_WIDTH and _why(N=513, rgba=8) == MANY_PLANES | ALIGNMENT


def test_the_three_queries_agree_on_fp32_expanded_mpis(lib):
    """gmpi_mpi_render_fwd_plan is _plan_ex of one MPI at the given rgba; _variant is _plan_ex of 2^20 views without a pointer."""
    why = ctypes.c_uint32(0)
    for v in ("auto", "direct", "staged"):
        with forced_kernel(v):
            for V, N, Wt, HW, rgba in itertools.product((1, 4), (16, 512, 513), (1020, 1022, 1024), (48, 300, 1024), (None, 8, 16)):
                plan = lib.gmpi_mpi_render_fwd_plan(V, N, 1024, Wt, HW, HW, rgba, ctypes.byref(why))
                case = (v, V, N, Wt, HW, rgba)
                assert (plan, why.value) == _lib.fwd_plan(_lib.make_desc(M=1, V=V, N=N, Ht=1024, Wt=Wt, H=HW, W=HW, rgba=rgba)), case
                staged = _lib.fwd_plan(_lib.make_desc(M=1, V=1 << 20, N=N, Ht=1024, Wt=Wt, H=HW, W=HW))[0] == _lib.PLAN_STAGED
                assert lib.gmpi_mpi_render_fwd_variant(N, 1024, Wt, HW, HW).decode() == \
                    ("fwd_staged_tma_64x30" if staged else "fwd_direct_32x8"), case


def test_warning_sees_every_mpi_tensor(lib, monkeypatch):
    """A factored MPI whose rgb, or bg_rgb, base is 8 bytes off a 16-byte boundary renders on the direct kernels: the wrapper warns."""
    monkeypatch.setattr(mpi, "_warned_direct", set())
    for ptrs in (dict(rgb=24, alpha=32, bg_rgb=48), dict(rgb=16, alpha=32, bg_rgb=56)):
        with pytest.warns(RuntimeWarning, match="MPI base pointer is not 16-byte aligned"):
            mpi._warn_if_direct(_lib.make_desc(**SIZES, **ptrs))
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        mpi._warn_if_direct(_lib.make_desc(**SIZES, rgb=16, alpha=32, bg_rgb=48))


def test_no_warning_for_the_alignment_of_a_tensor_copied_before_the_launch(lib, monkeypatch):
    """An fp64 MPI is rendered from a fresh fp32 copy, so the alignment of the caller's tensor does not matter."""
    monkeypatch.setattr(mpi, "_warned_direct", set())
    x = torch.rand(2 * 4 * 8 * 8 + 1, dtype=torch.float64)[1:].view(1, 2, 4, 8, 8)
    assert x.data_ptr() % 16 == 8
    launched, options = mpi._launch_mpi([x, None, None, None], 4, 1024, 1024, 0)
    assert launched[0].dtype == torch.float32 and launched[0].data_ptr() % 16 == 0
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        mpi._warn_if_direct(mpi._mpi_desc(launched, 4, 1024, 1024, options))
    with pytest.warns(RuntimeWarning, match="not 16-byte aligned"):
        mpi._warn_if_direct(mpi._mpi_desc([x, None, None, None], 4, 1024, 1024, 0))


# ------------------------------------------------------------------------------------------------------------------------------
# GPU: each launch takes the kernel its plan query predicts
# ------------------------------------------------------------------------------------------------------------------------------
MPI_PTRS = {"expanded": ("rgba",), "factored": ("rgb", "alpha"), "factored_bg": ("rgb", "alpha", "bg_rgb")}


def _launch_cases():
    """(form, fp16, case kwargs, expected why) per test id.  Default: 2 MPIs x 2 views of 256^2 (144 tiles), 8 planes of 64x64."""
    out = []
    for form, half in itertools.product(MPI_PTRS, (False, True)):
        cases = [("staged", {}, 0)]
        cases += [(f"misaligned_{k}", dict(misalign=k), ALIGNMENT) for k in MPI_PTRS[form]]
        cases += [("Wt66", dict(Wt=66), TEX_WIDTH), ("Wt68", dict(Wt=68), TEX_WIDTH if half else 0),
                  ("few_tiles", dict(img=64, views=1), FEW_TILES), ("N513", dict(N=513, tex=8), MANY_PLANES),
                  ("forced_direct", dict(variant="direct"), FORCED), ("forced_staged_few_tiles", dict(img=64, views=1, variant="staged"), 0)]
        out += [pytest.param(form, half, kw, why, id=f"{form}-{'fp16' if half else 'fp32'}-{name}") for name, kw, why in cases]
    return out


LAUNCH_CASES = _launch_cases()


def _render(form, half, N=8, tex=64, Wt=None, img=256, views=2, misalign=None, seed=5):
    """Descriptors (early stop at tau = 0, and off) of one render, and their colour/depth outputs."""
    dev = torch.device("cuda:0")
    case = synth.make_case(n_planes=N, tex=tex, img=img, n_mpi=2, views_per_mpi=views, seed=seed, rgba=False)
    geo = {k: getattr(case, k).to(dev) for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
    gen = torch.Generator().manual_seed(seed)
    hw = (tex, Wt or tex)
    rand = lambda *s: torch.rand(s, generator=gen).to(dev, torch.float16 if half else torch.float32)
    if form == "expanded":
        m = dict(rgba=rand(2, N, 4, *hw))
    else:
        m = dict(rgb=rand(2, 3, *hw), alpha=rand(2, N, 1, *hw), bg_rgb=rand(2, 3, *hw) if form == "factored_bg" else None)
    if misalign:
        m[misalign] = misaligned(m[misalign], 8)
    V, _, H, W = geo["ray_dir"].shape
    descs, outs = [], []
    for tau in (0.0, None):
        o = dict(color=torch.empty((V, 3, H, W), device=dev), depth=torch.empty((V, 1, H, W), device=dev),
                 flags=torch.zeros(1, dtype=torch.int32, device=dev))
        opts = _lib.OPT_ALIGN_CORNERS | (F16 if half else 0) | (_lib.OPT_EARLY_STOP if tau is not None else 0)
        descs.append(_lib.make_desc(options=opts, M=2, V=V, N=N, Ht=hw[0], Wt=hw[1], H=H, W=W, view_group=1, early_stop=tau,
                                    **geo, **m, **o))
        outs.append(o)
    return descs, outs, (m, geo)       # the tensors behind the descriptors' pointers


@pytest.mark.gpu
@pytest.mark.parametrize("form,half,kw,expect_why", LAUNCH_CASES)
def test_each_launch_takes_the_kernel_its_plan_predicts(form, half, kw, expect_why, lib):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    kw = dict(kw)
    with forced_kernel(kw.pop("variant", "auto")):
        (es, plain), (out_es, out_plain), keep = _render(form, half, **kw)
        plan, why = _lib.fwd_plan(es)
        assert why == expect_why and _lib.fwd_plan(plain) == (plan, why), (plan, why)
        _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(es)))
        skipped, total = early_stop_stats()
        stages = -(-es.W // 64) * -(-es.H // 30) * es.V * es.N
        assert total == (stages if plan == _lib.PLAN_STAGED else 0), (plan, why, total, stages)
        _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(plain)))
        torch.cuda.synchronize()
    for k in ("color", "depth", "flags"):
        assert_bitwise(out_es[k], out_plain[k], k)
