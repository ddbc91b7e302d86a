"""Each backward launches the kernel its plan predicts (gmpi_mpi_render_bwd_plan_ex; run on an H100: pytest -m gpu).

For the expanded, factored and factored + bg_rgb MPI, at the box kernel's shape and at every reason it may be refused, the test runs
the training forward (with its saved transmittance where the case has one), then gmpi_mpi_render_bwd_ex and
gmpi_mpi_render_bwd_deterministic_ex, reads the key of the kernel each launched (gmpi_debug_last_render_key), and checks it against
the plan: kKeyStaged exactly when the plan is GMPI_PLAN_STAGED, with the kKeyFac, kKeyDet and kKeyAC bits the call implies.  The
forward's key is checked against its own plan the same way, and every gradient against the oracle."""
import ctypes
import itertools

import numpy as np
import pytest
import torch

from conftest import rel_err
from ml_gmpi_b200 import _lib, expand_factored
from testlib import (EXPECT, FACTORED_RGB_EXPECT, GEOMETRY, KEY_AC, KEY_BWD, KEY_DET, KEY_EMIT, KEY_FAC, KEY_STAGED, check_factored, dev,
                     forced_kernel, lib, misaligned, on_device, oracle_backward, synth_case)

pytestmark = pytest.mark.gpu
FEW_TILES, FORCED = 2, 16
NO_TRANSMITTANCE, IMG_WIDTH, GRAD_ALIGNMENT = 32, 64, 128
GRADS = {"expanded": ("g_rgba",), "factored": ("g_rgb", "g_alpha"), "factored_bg": ("g_rgb", "g_alpha", "g_bg_rgb")}
# the gradient each form's "misaligned_gradient" case moves 8 bytes off a 16-byte boundary
MISALIGNED_GRAD = {"expanded": "g_rgba", "factored": "g_alpha", "factored_bg": "g_bg_rgb"}
# name: (case keywords, expected why).  Default: 2 MPIs x 2 views of 256^2 (144 forward tiles), 8 planes of 64^2.  W=66 / W=68: 512
# rows of a 512^2 image's first W columns (144 tiles).
CASES = {
    "staged": ({}, 0),
    "no_transmittance": (dict(transmittance=False), NO_TRANSMITTANCE),
    "W68": (dict(img=512, W=68), 0),
    "W66": (dict(img=512, W=66), IMG_WIDTH),
    "misaligned_gradient": (dict(misalign="gradient"), GRAD_ALIGNMENT),
    "misaligned_transmittance": (dict(misalign="transmittance"), GRAD_ALIGNMENT),
    "few_tiles": (dict(img=64, views=1), FEW_TILES),
    "forced_direct": (dict(variant="direct"), FORCED),
    "forced_staged_few_tiles": (dict(img=64, views=1, variant="staged"), 0),
}


def _last_key():
    key = ctypes.c_uint32(0)
    _lib.check(_lib.load().gmpi_debug_last_render_key(torch.cuda.current_device(), ctypes.byref(key)))
    return key.value


def _train(form, img=256, W=None, views=2, transmittance=True, misalign=None, seed=6):
    """The tensors of one training call -- a catalogue case (testlib.synth_case) like the transmittance and factored suites'
    "staged_shape": geometry, MPI whose background shows through, saved transmittance, upstream gradients -- and the forward's
    descriptor.  W: the image's first W columns."""
    d = dev()
    c = synth_case(n_planes=8, tex=64, img=img, n_mpi=2, views_per_mpi=views, seed=seed, alpha_scale=0.25, visible=True,
                   rays=(lambda r: r[..., :W].contiguous()) if W else None)
    geo = dict(zip(GEOMETRY, on_device(c, *GEOMETRY)))
    rgba, rgb, alpha, bg, gc, gd = on_device(c, "rgba", "rgb", "alpha", "bg", "gc", "gd")
    m = dict(rgba=rgba) if form == "expanded" else dict(rgb=rgb, alpha=alpha, bg_rgb=bg if form == "factored_bg" else None)
    V, _, H, Wi = geo["ray_dir"].shape
    t = torch.empty((V, 8, H, Wi), device=d) if transmittance else None
    if misalign == "transmittance":
        t = misaligned(t, 8)
    out = dict(color=torch.empty((V, 3, H, Wi), device=d), depth=torch.empty((V, 1, H, Wi), device=d),
               flags=torch.zeros(1, dtype=torch.int32, device=d))
    keep = dict(geo, **m, **out, transmittance=t, g_color=gc, g_depth=gd)
    desc = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS, M=2, V=V, N=8, Ht=64, Wt=64, H=H, W=Wi, view_group=1,
                          **{k: v for k, v in keep.items() if k not in ("g_color", "g_depth")})
    return desc, keep


def _grads(form, keep, misalign):
    """Gradient buffers of the MPI's form (filled with NaN: GMPI_ZERO_GRAD must overwrite them), one 8 bytes off a 16-byte boundary
    in the misaligned_gradient case."""
    src = {"g_rgba": "rgba", "g_rgb": "rgb", "g_alpha": "alpha", "g_bg_rgb": "bg_rgb"}
    out = {}
    for k in GRADS[form]:
        t = torch.full_like(keep[src[k]], float("nan"))
        out[k] = misaligned(t, 8) if misalign == "gradient" and k == MISALIGNED_GRAD[form] else t
    return out


def _backward_desc(form, keep, grads, desc):
    d = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_ZERO_GRAD, M=desc.M, V=desc.V, N=desc.N, Ht=desc.Ht, Wt=desc.Wt,
                       H=desc.H, W=desc.W, view_group=1, **{k: keep[k] for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir", "rgba",
                                                                                "rgb", "alpha", "bg_rgb", "transmittance", "g_color",
                                                                                "g_depth") if k in keep}, **grads)
    return d


def _check_gradients(form, keep, grads):
    """The gradients against the oracle's expanded gradient, within the parity bar (factored: d rgb sums N or N - 1 planes)."""
    if form == "expanded":
        rgba = keep["rgba"]
    else:
        rgba = expand_factored(keep["rgb"], keep["alpha"], keep["bg_rgb"])
    case = {k: keep[k] for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
    ref = oracle_backward(case, keep["g_color"], keep["g_depth"], rgba=rgba)
    got = {k: v.cpu().numpy() for k, v in grads.items()}
    if form == "expanded":
        e = rel_err(got["g_rgba"], ref)
        assert e <= EXPECT, e
    elif form == "factored_bg":
        check_factored((got["g_rgb"], got["g_alpha"], got["g_bg_rgb"]), ref)
    else:
        e = (rel_err(got["g_rgb"], ref[:, :, :3].astype(np.float64).sum(1)), rel_err(got["g_alpha"], ref[:, :, 3:4]))
        assert e[0] <= FACTORED_RGB_EXPECT and e[1] <= EXPECT, e


@pytest.mark.parametrize("form,name", list(itertools.product(GRADS, CASES)))
def test_each_backward_launches_the_kernel_its_plan_predicts(form, name, lib):
    kw, expect_why = CASES[name]
    kw = dict(kw)
    fac = KEY_FAC if form != "expanded" else 0
    with forced_kernel(kw.pop("variant", "auto")):
        fwd, keep = _train(form, **kw)
        fwd_plan, _ = _lib.fwd_plan(fwd)
        _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(fwd)))
        staged_fwd = KEY_STAGED | fac | (KEY_EMIT if keep["transmittance"] is not None else 0)
        assert _last_key() == KEY_AC | (staged_fwd if fwd_plan == _lib.PLAN_STAGED else 0), fwd_plan
        for det in (False, True):
            grads = _grads(form, keep, kw.get("misalign"))
            d = _backward_desc(form, keep, grads, fwd)
            plan, why = _lib.bwd_plan(d)
            assert why == expect_why and plan == (_lib.PLAN_STAGED if why == 0 else _lib.PLAN_DIRECT), (plan, why)
            if det:
                n = _lib.deterministic_scratch_bytes(d)
                scratch = torch.empty(n, dtype=torch.uint8, device=dev())
                _lib.check(lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), scratch.data_ptr(), n))
            else:
                _lib.check(lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)))
            key = _last_key()
            staged = KEY_STAGED | fac if plan == _lib.PLAN_STAGED else 0
            assert key == KEY_BWD | KEY_AC | (KEY_DET if det else 0) | staged, (det, plan, why, key)
            torch.cuda.synchronize()
            _check_gradients(form, keep, grads)
