"""The flag word (GMPI_FLAG_*) of every forward path against the CPU oracle, whose flag rule tests/test_oracle_golden.py pins to the
reference's verdicts (run on an H100: pytest -m gpu; test_wrong_flag_rules_disagree_with_the_oracle runs without a GPU).

The flags are how the library reports the reference's data-dependent asserts: alpha outside [0, 1] (mpi.py:185-187), a plane
behind view 0's eye (mpi.py:70, over the planes of the MPIs some view renders) and rays leaving the last plane (mpi.py:103-128,
where the reference calls sys.exit).  A wrong bit either stops a run the reference continues or lets one continue that the
reference stops, so every path must give the oracle's word exactly, with GMPI_CHECK_LAST_PLANE on and off:

  cases  the crafted edges of tests/golden/flags_edges.npz (|u| or |v| exactly 1 and one ulp beyond on the last plane, NaN ray,
         distance equal to view 0's eye z and one ulp below, a plane behind a later view's eye or in an MPI no view renders, NaN
         distance, alpha edges), reference fixtures, and variants built here the same way: a 4-MPI batch with views [0,0,1,3,3]
         (MPI 2 has none) of 37 x 70 pixels whose extreme pixel is at row 36, columns 64-69 (the edge of a partial 64 x 30 tile),
         and the same batch in the cam form (rays generated in the kernel; the edge from the rays gmpi_debug_cam_rays returns,
         view 0's eye from cam[13:16]);
  paths  the descriptor forward (expanded, factored with and without bg_rgb, native fp16 expanded and factored, early stop at
         tau = 1e-3 with every pixel opaque at plane 0, training with the saved transmittance, the uint8 video epilogue, the fused
         gather into one local buffer), the classic gmpi_mpi_render_fwd / _fwd_train / _fwd_gather, and the host entry points
         gmpi_mpi_render_fwd_host / gmpi_mpi_render_host_ex (with rays and with cam), each on the direct kernel and the staged
         kernel at a 2- and a 3-stage ring.

The range check (gmpi_mpi_check_range, _f16) equals mpi_oracle.check_range at its value edges on its vector and scalar kernels, and
MPI(validate=...) turns the flags into the reference's exceptions."""
import ctypes

import numpy as np
import pytest
import torch

import mpi_oracle
from conftest import load_golden
from ml_gmpi_b200 import _lib
from ml_gmpi_b200.mpi import MPI, MPIOutOfPlaneError
from ml_gmpi_b200.synth import ffhq_dhw, make_poses
from ml_gmpi_b200.camera import cam_params
from testlib import FLAG_CASES, FORWARD_FLAGS, dev, forced_kernel, kernel_fixture, oracle_forward

gpu = pytest.mark.gpu
OOB, BEHIND = mpi_oracle.FLAG_LAST_PLANE_OOB, mpi_oracle.FLAG_PLANE_BEHIND_EYE
OPT_AC, OPT_CHECK, OPT_M11, OPT_ES, OPT_F16 = (_lib.OPT_ALIGN_CORNERS, _lib.OPT_CHECK_LAST_PLANE, _lib.OPT_COLOR_MINUS1_1,
                                               _lib.OPT_EARLY_STOP, _lib.OPT_MPI_F16)
variant = kernel_fixture("direct", "staged2", "staged3")


# ------------------------------------------------------------------------------------------------------------------------------
# cases
# ------------------------------------------------------------------------------------------------------------------------------
def last_plane_xy(c):
    """(x, y) [V,H,W] of every ray at the last plane of its MPI, in the reference's fp32 op sequence (mpi.py:67-81)."""
    d = c["dhw"][c["view2mpi"], -1, 0][:, None, None]
    e = c["eye"][:, :, None, None]
    r = c["ray_dir"]
    with np.errstate(divide="ignore", invalid="ignore"):        # ray_z == 0: inf and NaN, as in the reference
        s = (d - e[:, 2]) / r[:, 2]
        return e[:, 0] + r[:, 0] * s, e[:, 1] + r[:, 1] * s


def pinned(c, axis, exact):
    """Copy of `c` whose last plane's width (axis "u") or height ("v") puts the pixel of largest |x| (|y|) exactly at |u| == 1
    (exact) or one ulp beyond; returns also that pixel (view, row, column)."""
    x, y = last_plane_xy(c)
    t = x if axis == "u" else y
    k = int(np.argmax(np.abs(t)))
    size = np.float32(2) * np.abs(t.flat[k])
    c = {key: np.array(val, copy=True) for key, val in c.items()}
    c["dhw"][:, -1, 2 if axis == "u" else 1] = size if exact else np.nextafter(size, np.float32(0))
    return c, np.unravel_index(k, t.shape)


def batch4(H=37, W=70, seed=7):
    """4 MPIs x 5 planes of 16^2, views [0,0,1,3,3] (MPI 2 has none) of H x W pixels cropped from a 70^2 image, and cam [V,16]."""
    yaws, pitches = [0.15, 0.3, -0.2, 0.25, -0.1], [0.05, 0.1, -0.08, 0.02, -0.12]
    ray, eye, z, c2w, _, _ = make_poses(5, 70, yaws=yaws, pitches=pitches)
    y0 = (70 - H) // 2
    c = dict(rgba=np.random.default_rng(seed).random((4, 5, 4, 16, 16), dtype=np.float32),
             dhw=np.broadcast_to(ffhq_dhw(5).numpy()[None], (4, 5, 3)).copy(), view2mpi=np.array([0, 0, 1, 3, 3], np.int32),
             ray_dir=ray[:, :, y0:y0 + H, :W].contiguous().numpy(), eye=eye.numpy(), z_dir=z.numpy(), align_corners=np.int32(1))
    return c, c2w


def _at_edge(c, comp):
    """Stretch ray component comp (0: x, 1: y) of view 4 at row 36, columns 64-69 3x: the extreme pixel moves there."""
    c = {k: np.array(v, copy=True) for k, v in c.items()}
    c["ray_dir"][4, comp, 36, 64:70] *= np.float32(3)
    return c


def _geometry_variants(c, eye0_z, eye1_z):
    """The plane-distance edges of a batch with view2mpi [0,0,1,3,3]."""
    out = {}
    for tag, m, i, d in (("viewless_behind", 2, 0, -0.5), ("viewless_nan", 2, 1, np.nan), ("behind_view1", 0, 0, (eye0_z + eye1_z) / 2),
                         ("eq_eye0", 3, 0, eye0_z), ("ulp_below_eye0", 3, 2, np.nextafter(eye0_z, np.float32(0)))):
        v = {k: np.array(val, copy=True) for k, val in c.items()}
        v["dhw"][m, i, 0] = d
        out[tag] = v
    return out


def build_cases():
    """name -> case (numpy) of every ray-form case: the fixture cases, reference fixtures, and the 4-MPI partial-tile batch."""
    cases = {name: c for name, _, c in FLAG_CASES}
    for name in ("tiny_2mpi_3view", "tiny_2mpi_3view_acfalse", "out_of_plane", "nonsquare", "alpha_one_planes", "magnify_40_from_16",
                 "edge_ragged_zero_views", "edge_odd_sizes", "edge_acfalse_nonsquare"):
        g = load_golden(name)
        cases[name] = {k: g[k] for k in ("rgba", "dhw", "view2mpi", "ray_dir", "eye", "z_dir", "align_corners")}
    b, _ = batch4()
    eye = b["eye"]
    assert eye[0, 2] > 0 and eye[1, 2] > eye[0, 2]
    cases["b4_clean"] = b
    cases.update({"b4_" + k: v for k, v in _geometry_variants(b, eye[0, 2], eye[1, 2]).items()})
    for axis, comp in (("u", 0), ("v", 1)):
        for exact in (True, False):
            c, (v, row, col) = pinned(_at_edge(b, comp), axis, exact)
            assert (v, row) == (4, 36) and 64 <= col <= 69, (axis, v, row, col)
            cases[f"b4_edge_{axis}_{'exact' if exact else 'ulp'}"] = c
    return cases


_CASES = None
_CAM_CASES = None


def cases():
    global _CASES
    if _CASES is None:
        _CASES = build_cases()
    return _CASES


def cam_cases():
    """name -> case of the cam form: the 4-MPI batch's cam [V,16]; ray_dir, eye and z_dir are what the kernel derives from it
    (the rays of gmpi_debug_cam_rays, eye = cam[13:16], z = the rotation's third column), so the oracle sees the kernel's rays."""
    global _CAM_CASES
    if _CAM_CASES is None:
        b, c2w = batch4()
        V, _, H, W = b["ray_dir"].shape
        cam = cam_params(c2w, 1.1 * W, H, W).to(dev())
        rays = torch.empty((V, 3, H, W), device=dev())
        _lib.check(_lib.load().gmpi_debug_cam_rays(cam.data_ptr(), rays.data_ptr(), V, H, W, None))
        torch.cuda.synchronize()
        camn = cam.cpu().numpy()
        b = dict(b, cam=camn, ray_dir=rays.cpu().numpy(), eye=np.ascontiguousarray(camn[:, 13:16]),
                 z_dir=np.ascontiguousarray(camn[:, 4:13].reshape(V, 3, 3)[:, :, 2]))
        eye = b["eye"]
        assert eye[0, 2] > 0 and eye[1, 2] > eye[0, 2]
        out = {"cam_clean": b}
        out.update({"cam_" + k: v for k, v in _geometry_variants(b, eye[0, 2], eye[1, 2]).items()})
        for exact in (True, False):         # the edge of the whole batch: the width from the kernel's own rays
            out[f"cam_edge_u_{'exact' if exact else 'ulp'}"] = pinned(b, "u", exact)[0]
        _CAM_CASES = out
    return _CAM_CASES


def oracle_flags(c, check):
    return oracle_forward(c, align_corners=bool(c["align_corners"]), check_last_plane=check)[2]


def test_built_cases_sit_on_their_edges():
    """The premise of the variants built here, on the oracle: the exact edges pass, one ulp beyond is out of the last plane, the
    distance edges flag exactly as the reference's rule says (only view 0's eye, only rendered MPIs, equality passes, NaN fails)."""
    want = {"b4_clean": 0, "b4_viewless_behind": 0, "b4_viewless_nan": 0, "b4_behind_view1": 0, "b4_eq_eye0": 0,
            "b4_ulp_below_eye0": BEHIND, "b4_edge_u_exact": 0, "b4_edge_u_ulp": OOB, "b4_edge_v_exact": 0, "b4_edge_v_ulp": OOB}
    cs = cases()
    for name, f in want.items():
        assert oracle_flags(cs[name], True) == f, name


# ------------------------------------------------------------------------------------------------------------------------------
# paths
# ------------------------------------------------------------------------------------------------------------------------------
def _stream():
    return torch.cuda.current_stream().cuda_stream


def _device_inputs(c, path):
    """Descriptor fields of case `c` (device tensors) for a path: the MPI form, the camera form, options."""
    d = dev()
    rgba = torch.from_numpy(np.ascontiguousarray(c["rgba"])).to(d)
    if path == "early_stop":
        rgba = rgba.clone()
        rgba[:, 0, 3] = 1.0                      # every pixel is opaque at plane 0: it stops long before the last plane
    half = path.startswith("f16")
    dt = torch.float16 if half else torch.float32
    if "factored" in path:
        mpi = dict(rgb=rgba[:, 0, :3].contiguous().to(dt), alpha=rgba[:, :, 3:4].contiguous().to(dt),
                   bg_rgb=None if path.endswith("nobg") else rgba[:, -1, :3].contiguous().to(dt))
    else:
        mpi = dict(rgba=rgba.to(dt))
    if "cam" in c:
        cams = dict(cam=torch.from_numpy(c["cam"]).to(d))
    else:
        cams = {k: torch.from_numpy(np.ascontiguousarray(c[k])).to(d) for k in ("ray_dir", "eye", "z_dir")}
    M, N, _, Ht, Wt = c["rgba"].shape
    V, _, H, W = c["ray_dir"].shape
    opts = (OPT_AC if c["align_corners"] else 0) | (OPT_F16 if half else 0) | (OPT_ES if path == "early_stop" else 0)
    return dict(options=opts, M=M, V=V, N=N, Ht=Ht, Wt=Wt, H=H, W=W, early_stop=1e-3 if path == "early_stop" else None,
                view2mpi=torch.from_numpy(c["view2mpi"]).to(d), dhw=torch.from_numpy(np.ascontiguousarray(c["dhw"])).to(d), **mpi, **cams)


def _desc_fwd(i, **out):
    flags = torch.zeros(1, dtype=torch.int32, device=dev())
    _lib.check(_lib.load().gmpi_mpi_render_fwd_ex(ctypes.byref(_lib.make_desc(**i, **out, flags=flags, stream=_stream()))))
    torch.cuda.synchronize()
    return int(flags.item()) & 0xFFFFFFFF


def _outputs(i):
    V, H, W = i["V"], i["H"], i["W"]
    return dict(color=torch.empty((V, 3, H, W), device=dev()), depth=torch.empty((V, 1, H, W), device=dev()))


def _host_ex(i):
    """gmpi_mpi_render_host_ex from host copies of the inputs (MPI by MPI through the staging slots)."""
    h = {k: (v.cpu().contiguous() if torch.is_tensor(v) else v) for k, v in i.items()}
    V, H, W = i["V"], i["H"], i["W"]
    color, depth = torch.empty((V, 3, H, W)), torch.empty((V, 1, H, W))
    flags = np.zeros(1, np.uint32)
    d = _lib.make_desc(**h, color=color, depth=depth, flags=flags.ctypes.data)
    _lib.check(_lib.load().gmpi_mpi_render_host_ex(ctypes.byref(d), 0))
    return int(flags[0])


def run_path(path, c, check):
    """Flag word of one forward of case `c` through `path`."""
    lib = _lib.load()
    i = _device_inputs(c, path)
    if check:
        i["options"] |= OPT_CHECK
    V, H, W, N = i["V"], i["H"], i["W"], i["N"]
    if path in ("expanded", "factored_bg", "factored_nobg", "f16", "f16_factored", "early_stop"):
        return _desc_fwd(i, **_outputs(i))
    if path == "train":
        return _desc_fwd(i, **_outputs(i), transmittance=torch.empty((V, N, H, W), device=dev()))
    if path == "video":
        i["options"] |= OPT_M11
        return _desc_fwd(i, video_rgb=torch.empty((V, H, W, 3), dtype=torch.uint8, device=dev()),
                         video_depth=torch.empty((V, H, W, 1), dtype=torch.uint8, device=dev()), depth_near=0.9, depth_range=0.3)
    if path == "gather":
        buf = torch.empty((V, 4, H, W), device=dev())
        ptrs = torch.tensor([buf.data_ptr()], dtype=torch.int64, device=dev())
        return _desc_fwd(i, peer_frames=ptrs, n_peers=1, frame_offset=0)
    if path == "host_ex":
        return _host_ex(i)
    flags = torch.zeros(1, dtype=torch.int32, device=dev())
    p = [i[k].data_ptr() for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")]
    sizes = (i["M"], V, N, i["Ht"], i["Wt"], H, W)
    o = _outputs(i)
    if path == "classic_fwd":
        rc = lib.gmpi_mpi_render_fwd(*p, o["color"].data_ptr(), o["depth"].data_ptr(), flags.data_ptr(), *sizes, i["options"], _stream())
    elif path == "classic_train":
        t = torch.empty((V, N, H, W), device=dev())
        rc = lib.gmpi_mpi_render_fwd_train(*p, o["color"].data_ptr(), o["depth"].data_ptr(), t.data_ptr(), flags.data_ptr(), *sizes,
                                           i["options"], _stream())
    elif path == "classic_gather":
        buf = torch.empty((V, 4, H, W), device=dev())
        ptrs = torch.tensor([buf.data_ptr()], dtype=torch.int64, device=dev())
        rc = lib.gmpi_mpi_render_fwd_gather(*p, ptrs.data_ptr(), 1, 0, flags.data_ptr(), *sizes, i["options"], _stream())
    elif path == "host_fwd":
        h = [np.ascontiguousarray(c[k]) for k in ("rgba", "view2mpi", "dhw", "ray_dir", "eye", "z_dir")]
        color, depth = np.empty((V, 3, H, W), np.float32), np.empty((V, 1, H, W), np.float32)
        hf = np.zeros(1, np.uint32)
        _lib.check(lib.gmpi_mpi_render_fwd_host(*[a.ctypes.data for a in h], color.ctypes.data, depth.ctypes.data, hf.ctypes.data,
                                                *sizes, i["options"], 0))
        return int(hf[0])
    else:
        raise AssertionError(path)
    _lib.check(rc)
    torch.cuda.synchronize()
    return int(flags.item()) & 0xFFFFFFFF


PATHS = ["expanded", "factored_bg", "factored_nobg", "f16", "f16_factored", "early_stop", "train", "video", "gather",
         "classic_fwd", "classic_train", "classic_gather", "host_fwd", "host_ex"]
CAM_PATHS = ["expanded", "factored_bg", "f16", "f16_factored", "early_stop", "video", "gather", "host_ex"]


@gpu
@pytest.mark.parametrize("path", PATHS)
def test_flag_word_of_every_forward_path_equals_the_oracle(path, variant):
    bad = []
    all_cases = dict(cases())
    if path in CAM_PATHS:
        all_cases.update(cam_cases())
    for name, c in all_cases.items():
        for check in (True, False):
            got, want = run_path(path, c, check), oracle_flags(c, check)
            if got != want:
                bad.append((name, "check" if check else "nocheck", got, want))
    assert not bad, (path, variant, bad)
    if path == "host_ex":
        _lib.check(_lib.load().gmpi_mpi_release_host_cache())


# ------------------------------------------------------------------------------------------------------------------------------
# range flags
# ------------------------------------------------------------------------------------------------------------------------------
VALUES32 = {"one": 1.0, "next_above_one": float(np.nextafter(np.float32(1), np.float32(2))), "zero": 0.0, "neg_zero": -0.0,
            "neg_denormal": -float(np.float32(2.0 ** -149)), "inf": np.inf, "neg_inf": -np.inf, "nan": np.nan}
VALUES16 = dict(VALUES32, next_above_one=1.0 + 2.0 ** -10, neg_denormal=-(2.0 ** -24))


def _range_layouts(kernel):
    """(M, N, Ht, Wt, byte offset of the base) of the vector kernel, or of the scalar one forced by the slab or by the base."""
    return {"vector": (2, 3, 8, 16, 0), "scalar_slab": (2, 3, 5, 7, 0), "scalar_offset": (2, 3, 8, 16, 8)}[kernel]


@gpu
@pytest.mark.parametrize("dtype", ["f32", "f16"])
@pytest.mark.parametrize("kernel", ["vector", "scalar_slab", "scalar_offset"])
def test_range_flags_equal_the_oracle_at_their_value_edges(kernel, dtype):
    lib = _lib.load()
    M, N, Ht, Wt, off = _range_layouts(kernel)
    dt, np_dt = (torch.float16, np.float16) if dtype == "f16" else (torch.float32, np.float32)
    check = lib.gmpi_mpi_check_range_f16 if dtype == "f16" else lib.gmpi_mpi_check_range
    n = M * N * 4 * Ht * Wt
    esz = 2 if dtype == "f16" else 4
    buf = torch.empty(n + 16 // esz, dtype=dt, device=dev())
    base = np.random.default_rng(3).random((M, N, 4, Ht, Wt)).astype(np_dt) * np_dt(0.999)
    slab = Ht * Wt
    positions = {"first": 0, "last": n - 1, "slab_tail": 5 * slab - 1,                  # slab 4 = MPI 0, plane 1, red
                 "last_mpi_colour": ((M - 1) * N * 4 + (N - 1) * 4 + 1) * slab + slab // 2,
                 "last_mpi_alpha": ((M - 1) * N * 4 + (N - 1) * 4 + 3) * slab + slab // 3}
    bad = []
    for vname, val in (VALUES16 if dtype == "f16" else VALUES32).items():
        for pname, pos in positions.items():
            x = base.copy()
            x.reshape(-1)[pos] = np_dt(val)
            view = buf[off // esz: off // esz + n]
            view.copy_(torch.from_numpy(x.reshape(-1)).to(dev()))
            flags = torch.zeros(1, dtype=torch.int32, device=dev())
            _lib.check(check(view.data_ptr(), M, N, Ht, Wt, flags.data_ptr(), _stream()))
            torch.cuda.synchronize()
            got, want = int(flags.item()), mpi_oracle.check_range(x.astype(np.float32))
            if got != want:
                bad.append((vname, pname, got, want))
    assert not bad, bad


# ------------------------------------------------------------------------------------------------------------------------------
# MPI(validate=...) raises what the reference raises
# ------------------------------------------------------------------------------------------------------------------------------
def _mpi_call(module, c):
    d = dev()
    v2m = c["view2mpi"]
    sel = [np.nonzero(v2m == m)[0] for m in range(c["rgba"].shape[0])]
    g = lambda a: [torch.from_numpy(np.ascontiguousarray(a[s])).to(d) for s in sel]     # noqa: E731
    return module(batch_rgba=torch.from_numpy(c["rgba"]).to(d), batch_dhw=torch.from_numpy(c["dhw"]).to(d), batch_ray_dir=g(c["ray_dir"]),
                  batch_eye_pos=g(c["eye"]), batch_z_dir=g(c["z_dir"]), separate_background=None, assert_not_out_of_last_plane=True)


# the reference's exception and message per verdict; where the reference calls sys.exit(1) the library raises instead
EXCEPTIONS = {"alpha": (AssertionError, "Expected alpha to be within the the range [0, 1]"),
              "behind-eye": (AssertionError, "Camera must be placed closer to origin than MPI."),
              "out-of-plane": (MPIOutOfPlaneError, "Ray's U/V direction goes out of plane")}


@gpu
@pytest.mark.parametrize("kernel", ["direct", "staged2"])
def test_mpi_module_raises_the_reference_exception_for_each_verdict(kernel):
    with forced_kernel(kernel):
        for name, verdict, c in FLAG_CASES:
            full = MPI(align_corners=bool(c["align_corners"]), validate="full")
            if verdict == "ok":
                _mpi_call(full, c)
            else:
                cls, msg = EXCEPTIONS[verdict]
                with pytest.raises(AssertionError) as e:
                    _mpi_call(full, c)
                assert type(e.value) is cls and str(e.value).startswith(msg), (name, e.value)
            defer = MPI(align_corners=bool(c["align_corners"]), validate="defer")
            _mpi_call(defer, c)                             # nothing is raised before raise_if_flagged
            if verdict in ("behind-eye", "out-of-plane"):
                cls, msg = EXCEPTIONS[verdict]
                with pytest.raises(AssertionError) as e:
                    defer.raise_if_flagged()
                assert type(e.value) is cls and str(e.value).startswith(msg), (name, e.value)
            else:
                defer.raise_if_flagged()                    # "defer" scans no alpha
            off = MPI(align_corners=bool(c["align_corners"]), validate="off")
            _mpi_call(off, c)
            assert off.last_flags() == FORWARD_FLAGS[verdict] & ~OOB, (name, off.last_flags())


# ------------------------------------------------------------------------------------------------------------------------------
# teeth: the plausible wrong rules each disagree with the oracle on some case (CPU)
# ------------------------------------------------------------------------------------------------------------------------------
def rule_flags(c, check, own_eye=False, all_mpis=False, strict_eye=False, strict_uv=False, nan_passes=False, every_plane=False):
    """The flag word in numpy, from the reference's fp32 coordinates, under the right rule or one of the wrong ones."""
    v2m, dhw, eye = c["view2mpi"], c["dhw"], c["eye"]
    flags = 0
    rendered = range(dhw.shape[0]) if all_mpis else sorted(set(v2m.tolist()))
    for m in rendered:
        views = np.nonzero(v2m == m)[0] if own_eye else [0]
        for v in views:
            d, ez = dhw[m, :, 0], eye[v, 2]
            bad = (d < ez) if nan_passes else ~(d > ez) if strict_eye else ~(d >= ez)
            if bad.any():
                flags |= BEHIND
    if check:
        planes = range(dhw.shape[1]) if every_plane else [dhw.shape[1] - 1]
        for i in planes:
            d = {k: np.array(v) for k, v in c.items()}
            d["dhw"] = dhw[:, [i] * dhw.shape[1]]
            x, y = last_plane_xy(d)
            u = np.float32(2) * x / dhw[v2m, i, 2][:, None, None]
            w = np.float32(2) * y / dhw[v2m, i, 1][:, None, None]
            for t in (u, w):
                if nan_passes:
                    out = (t > 1) | (t < -1)
                elif strict_uv:
                    out = ~((t > -1) & (t < 1))
                else:
                    out = ~((t >= -1) & (t <= 1))
                if out.any():
                    flags |= OOB
    return flags


WRONG_RULES = {"each view's own eye": dict(own_eye=True), "all MPIs, not the rendered ones": dict(all_mpis=True),
               "> for >=": dict(strict_eye=True), "< for <=": dict(strict_uv=True), "NaN passes": dict(nan_passes=True),
               "every plane, not the last": dict(every_plane=True)}


def test_wrong_flag_rules_disagree_with_the_oracle():
    """The right rule in numpy equals the oracle on every crafted case; each wrong rule differs from it on at least one, so a
    kernel that implemented it would fail test_flag_word_of_every_forward_path_equals_the_oracle."""
    cs = cases()
    for name, c in cs.items():
        for check in (True, False):
            assert rule_flags(c, check) == oracle_flags(c, check), (name, check)
    for rule, kw in WRONG_RULES.items():
        caught = [name for name, c in cs.items() for check in (True, False) if rule_flags(c, check, **kw) != oracle_flags(c, check)]
        assert caught, rule
