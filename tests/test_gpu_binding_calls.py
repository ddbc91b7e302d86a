"""The exact C calls the Python wrappers make, against a record (tests/golden/binding_calls.json).

The output tests cannot see options that leave the output unchanged: the view group, which entry point a render takes (skipping,
deterministic), the MPI base alignment (which decides staged against direct) or the direct-kernel warning.  Here the loaded library
is replaced by a proxy that records every gmpi_* call before it forwards it: the function, every scalar field of a descriptor, each
pointer as the caller's tensor it equals (or null, or `other` and its address mod 16), whether the stream is the current one, the
size arguments, and the RuntimeWarnings the wrapper call emits.

    python tests/test_gpu_binding_calls.py --record   # rewrites tests/golden/binding_calls.json (needs a GPU)
"""
import ctypes
import json
import os
import sys
import warnings

import pytest
import torch

from conftest import GOLDEN     # first: it puts the repository on sys.path when this file runs as a script
import ml_gmpi_b200 as g  # noqa: E402
from ml_gmpi_b200 import _lib, mpi, synth  # noqa: E402
from ml_gmpi_b200.camera import cam_params, focal_from_fov  # noqa: E402
from testlib import dev, misaligned  # noqa: E402

CALLS = os.path.join(GOLDEN, "binding_calls.json")


class _Recorder:
    """The loaded library, with every gmpi_* call recorded (its arguments as they are at the call) and then forwarded."""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)
        if not name.startswith("gmpi_"):
            return fn

        def call(*args):
            stream = torch.cuda.current_stream().cuda_stream
            self.calls.append((name, [_capture(a, t) for a, t in zip(args, fn.argtypes)], stream))
            return fn(*args)
        return call


def _capture(arg, argtype):
    if type(arg).__name__ == "CArgObject":                  # ctypes.byref(x)
        obj = arg._obj
        if isinstance(obj, _lib.RenderDesc):
            return ("desc", {f: getattr(obj, f) for f, _ in _lib.RenderDesc._fields_})
        return ("byref", type(obj).__name__)
    return ("ptr" if argtype is ctypes.c_void_p else "value", arg)


def _resolve(calls, names):
    """The recorded calls with every pointer replaced by the name of the tensor it equals, `stream` when it is the stream that was
    current at the call, null, or `other` and its address mod 16."""
    by_ptr = {}
    for n, t in names.items():
        if isinstance(t, torch.Tensor):
            by_ptr.setdefault(t.data_ptr(), n)

    def ptr(p, stream):
        if not p:
            return None
        if p == stream:
            return "stream"
        return by_ptr.get(p, f"other%16={p % 16}")

    out = []
    for name, args, stream in calls:
        rec = []
        for kind, a in args:
            if kind == "desc":
                a = {f: ptr(v, stream) if t is ctypes.c_void_p else v for (f, t), v in zip(_lib.RenderDesc._fields_, a.values())}
            elif kind == "ptr":
                a = ptr(a, stream)
            rec.append({kind: a})
        out.append([name] + rec)
    return out


def _geo(views=2, img=256):
    c = synth.make_case(n_planes=8, tex=8, img=img, n_mpi=2, views_per_mpi=views, seed=3, rgba=False)
    return {k: getattr(c, k).to(dev()) for k in ("dhw", "view2mpi", "ray_dir", "eye", "z_dir", "c2w")}


def _rand(*shape, dtype=torch.float32, seed=1):
    return torch.rand(shape, generator=torch.Generator().manual_seed(seed)).to(dev(), dtype)


def _views(names, **kw):
    """(inputs, call) of render_views on names' rgba and geometry."""
    def call():
        c, d = g.render_views(names["rgba"], names["dhw"], names["view2mpi"], names["ray_dir"], names["eye"], names["z_dir"], **kw)
        return dict(color=c, depth=d)
    return names, call


def _expanded(dtype=torch.float32, Wt=64, views=2, **kw):
    return _views(dict(_geo(views), rgba=_rand(2, 8, 4, 64, Wt, dtype=dtype)), **kw)


def _factored(dtype=torch.float32, bg=True, grad=False, **kw):
    names = dict(_geo(), rgb=_rand(2, 3, 64, 64, dtype=dtype, seed=2), alpha=_rand(2, 8, 1, 64, 64, dtype=dtype, seed=3),
                 bg_rgb=_rand(2, 3, 64, 64, dtype=dtype, seed=4) if bg else None)

    def call():
        for k in ("rgb", "alpha", "bg_rgb"):
            if grad and names[k] is not None:
                names[k].requires_grad_(True)
        c, d = g.render_views_factored(names["rgb"], names["alpha"], names["dhw"], names["view2mpi"], names["ray_dir"], names["eye"],
                                       names["z_dir"], bg_rgb=names["bg_rgb"], **kw)
        out = dict(color=c, depth=d)
        if grad:
            _backward(c, d)
            out.update({f"grad_{k}": names[k].grad for k in ("rgb", "alpha", "bg_rgb") if names[k] is not None})
        return out
    return names, call


def _backward(color, depth):
    gen = torch.Generator().manual_seed(9)
    gc, gd = torch.randn(color.shape, generator=gen).to(dev()), torch.randn(depth.shape, generator=gen).to(dev())
    ((color * gc).sum() + (depth * gd).sum()).backward()


def _train(deterministic=None, torch_switch=False):
    names = dict(_geo(), rgba=_rand(2, 8, 4, 64, 64).requires_grad_(True))

    def call():
        prev = torch.are_deterministic_algorithms_enabled()
        torch.use_deterministic_algorithms(torch_switch)
        try:
            c, d = g.render_views(names["rgba"], names["dhw"], names["view2mpi"], names["ray_dir"], names["eye"], names["z_dir"],
                                  deterministic=deterministic)
            _backward(c, d)
        finally:
            torch.use_deterministic_algorithms(prev)
        return dict(color=c, depth=d, grad_rgba=names["rgba"].grad)
    return names, call


def _reused_occupancy():
    names = dict(_geo(), rgba=_rand(2, 8, 4, 64, 64))

    def call():
        occ = g.build_occupancy(rgba=names["rgba"])
        c, d = g.render_views(names["rgba"], names["dhw"], names["view2mpi"], names["ray_dir"], names["eye"], names["z_dir"],
                              skip_empty=occ)
        return dict(occupancy=occ.occ, color=c, depth=d)
    return names, call


def _frames(cam=False, factored=False, video=None, **kw):
    geo = _geo()
    names = dict(geo, rgba=None if factored else _rand(2, 8, 4, 64, 64))
    if factored:
        names.update(rgb=_rand(2, 3, 64, 64, seed=2), alpha=_rand(2, 8, 1, 64, 64, seed=3), bg_rgb=_rand(2, 3, 64, 64, seed=4))
    rays = dict(ray_dir=geo["ray_dir"], eye=geo["eye"], z_dir=geo["z_dir"])
    if cam:
        names["cam"] = cam_params(geo["c2w"].cpu(), focal_from_fov(12.6, 256), 256, 256).to(dev())
        rays = dict(cam=names["cam"], H=256, W=256)

    def call():
        mpi_kw = {k: names[k] for k in ("rgba", "rgb", "alpha", "bg_rgb") if names.get(k) is not None}
        a, b = g.render_frames(dhw=names["dhw"], view2mpi=names["view2mpi"], video=video, **mpi_kw, **rays, **kw)
        return dict(frame_a=a, frame_b=b)
    return names, call


def _module(validate="full", skip_empty=False):
    geo = _geo()
    names = dict(geo, rgba=_rand(2, 8, 4, 64, 64))
    idx = [[0, 1], [2, 3]]

    def call():
        m = g.MPI(validate=validate, skip_empty=skip_empty)
        c, d = m(batch_rgba=names["rgba"], batch_dhw=names["dhw"], batch_ray_dir=[geo["ray_dir"][i] for i in idx],
                 batch_eye_pos=[geo["eye"][i] for i in idx], batch_z_dir=[geo["z_dir"][i] for i in idx], separate_background=None)
        return dict(color=c, depth=d, flags=m._flags)
    return names, call


def _renderer():
    from ml_gmpi_b200.renderer import MPIRenderer
    r = MPIRenderer(n_mpi_planes=8, plane_min_d=0.95, plane_max_d=1.12, plan_spatial_enlarge_factor=1.001,
                    plane_distances_sample_method="inverse", cam_fov=12.6, sphere_center_z=1.0, sphere_r=1.0,
                    horizontal_mean=0.0, horizontal_std=0.289, vertical_mean=0.0, vertical_std=0.127,
                    cam_pose_n_truncated_stds=2, cam_sample_method="truncated_gaussian", device=dev())
    r.set_cam(12.6, 128, 128)
    names = dict(rgba=_rand(4, 8, 4, 64, 64))
    yaws, pitches = torch.tensor([[0.1], [-0.1], [0.05], [0.0]]), torch.tensor([[0.05], [0.0], [-0.05], [0.02]])

    def call():
        img, depth, _, _ = r.render(names["rgba"], 128, 128, given_yaws=yaws, given_pitches=pitches)
        return dict(color=img, depth=depth)
    return names, call


CASES = {
    "views_fp32": lambda: _expanded(),
    "views_fp16_native": lambda: _expanded(torch.float16),
    "views_fp16_upcast": lambda: _expanded(torch.float16, Wt=68),          # Wt % 8 != 0: the fp16 plan is not the fp32 plan
    "views_fp64": lambda: _expanded(torch.float64),
    "views_misaligned": lambda: _views(dict(_geo(), rgba=misaligned(_rand(2, 8, 4, 64, 64), 8))),
    "views_align_corners_false": lambda: _expanded(align_corners=False),
    "views_check_last_plane": lambda: _expanded(check_last_plane=True),
    "views_color_minus1_1": lambda: _expanded(color_minus1_1=True),
    "views_view_group3": lambda: _expanded(views=3, view_group=3),
    "views_early_stop": lambda: _expanded(early_stop=0.05),
    "views_skip_empty": lambda: _expanded(skip_empty=True),
    "views_reused_occupancy": _reused_occupancy,
    "factored_fp32": lambda: _factored(),
    "factored_fp32_no_bg": lambda: _factored(bg=False),
    "factored_fp16": lambda: _factored(torch.float16),
    "factored_fp16_no_bg": lambda: _factored(torch.float16, bg=False),
    "factored_backward": lambda: _factored(grad=True),
    "backward": lambda: _train(),
    "backward_deterministic": lambda: _train(deterministic=True),
    "backward_torch_switch": lambda: _train(torch_switch=True),
    "frames_rays": lambda: _frames(),
    "frames_cam": lambda: _frames(cam=True, check_last_plane=True),
    "frames_video": lambda: _frames(video={"near": 0.88, "far": 1.12}, view_group=2),
    "frames_video_no_depth": lambda: _frames(video={"near": 0.88, "far": 1.12, "depth": False}),
    "frames_u8_round": lambda: _frames(video={"near": 0.88, "far": 1.12, "depth": False}, u8_round=True),
    "frames_factored": lambda: _frames(factored=True, early_stop=0.05),
    "frames_skip_empty": lambda: _frames(skip_empty=True),
    "mpi_validate_full": lambda: _module("full"),
    "mpi_validate_defer": lambda: _module("defer"),
    "mpi_validate_off": lambda: _module("off"),
    "mpi_skip_empty": lambda: _module("full", skip_empty=True),
    "renderer": _renderer,
}


def record(case, monkeypatch):
    """{calls, warnings} of one case, run on a side stream (so that `stream` is not the null default stream)."""
    names, call = CASES[case]()
    rec = _Recorder(_lib.load())
    monkeypatch.setattr(_lib, "_lib", rec)
    monkeypatch.setattr(mpi, "_warned_direct", set())
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with warnings.catch_warnings(record=True) as caught, torch.cuda.stream(s):
        warnings.simplefilter("always")
        outs = call()
    torch.cuda.synchronize()
    monkeypatch.undo()
    return {"calls": _resolve(rec.calls, {**names, **outs}),
            "warnings": [str(w.message) for w in caught if issubclass(w.category, RuntimeWarning)]}


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(CASES))
def test_wrappers_make_the_recorded_calls(case, monkeypatch):
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    g.build_library()
    with open(CALLS) as f:
        want = json.load(f)[case]
    assert json.loads(json.dumps(record(case, monkeypatch))) == want


if __name__ == "__main__" and "--record" in sys.argv:
    g.build_library()
    with pytest.MonkeyPatch.context() as mp:
        recs = {case: record(case, mp) for case in CASES}
    with open(CALLS, "w") as f:
        json.dump(recs, f, indent=1)
        f.write("\n")
    print(f"wrote {CALLS}: {sum(len(r['calls']) for r in recs.values())} calls in {len(recs)} cases")
