"""Flag-rule fixture for the ORACLE (tests/test_oracle_golden.py): small crafted cases and the verdict of the UNMODIFIED reference's
MPI.forward(..., assert_not_out_of_last_plane=True) on each, produced on CPU:

    python oracle/make_golden_flags.py      # needs /root/reference; writes tests/golden/flags_edges.npz

The reference reports its data-dependent checks by raising on the first one that fails:
  alpha        AssertionError "Expected alpha to be within ..."       (check_shapes, mpi.py:185-187)
  behind-eye   AssertionError "Camera must be placed closer ..."      (homography, mpi.py:70: every rendered plane vs view 0's eye z)
  out-of-plane SystemExit                                              (homography, mpi.py:103-128: last plane, |u| or |v| > 1 or NaN)
so every case breaks at most one of them.  Base batch: 3 MPIs x 5 planes, 16^2 textures, 4 views of 16^2 pixels with
view2mpi = [0, 0, 2, 2] (MPI 1 has no view).  The width / height of the last plane of the *_exact cases is exactly 2x (2y) of the
pixel with the largest |x| (|y|) at the last plane, computed with the reference's fp32 op sequence, so that pixel has |u| == 1;
the *_ulp cases take the next float below it, so |u| > 1.  The generator checks its own premise: each case gets the verdict it
was built for.  nonsquare / tiny_2mpi_3view_acfalse: the reference's verdict on those fixtures (their stored inputs).

Layout: names [K] and verdicts [K] (str); per case <name>__rgba = [seed] or [seed, m, i, c, y, x] (the MPI is rand_rgba(seed) with
element (m, i, c, y, x) set to <name>__rgba_value; shape <name>__rgba_shape) and <name>__{dhw, view2mpi, ray_dir, eye, z_dir, align_corners} = index j of
the array pool_j (cases share most arrays); fixtures [2] and fixture_verdicts [2].

TEST INFRASTRUCTURE ONLY.
"""
import contextlib
import io
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import ref_shim  # noqa: E402
from make_golden import OUT, cams, make_renderer, rand_rgba, save  # noqa: E402

VIEW2MPI = [0, 0, 2, 2]
M, N, TEX, IMG = 3, 5, 16, 16


def verdict(ref_mpi, c):
    """The reference's verdict on case `c` (packed arrays): which of its checks stops MPI.forward, or "ok"."""
    v2m = c["view2mpi"]
    sel = [np.nonzero(v2m == m)[0] for m in range(c["rgba"].shape[0])]
    g = lambda a: [torch.from_numpy(a[i]) for i in sel]        # noqa: E731
    mod = ref_mpi.MPI(align_corners=bool(c["align_corners"]))
    try:
        with contextlib.redirect_stdout(io.StringIO()), contextlib.redirect_stderr(io.StringIO()), torch.no_grad():
            mod(batch_rgba=torch.from_numpy(c["rgba"]), batch_dhw=torch.from_numpy(c["dhw"]), batch_ray_dir=g(c["ray_dir"]),
                batch_eye_pos=g(c["eye"]), batch_z_dir=g(c["z_dir"]), separate_background=None, assert_not_out_of_last_plane=True)
    except SystemExit:
        return "out-of-plane"
    except AssertionError as e:
        msg = str(e)
        if msg.startswith("Expected alpha"):
            return "alpha"
        if msg.startswith("Camera must be placed closer"):
            return "behind-eye"
        raise
    return "ok"


def last_plane_xy(c):
    """(x, y) [V,H,W] of every ray at the last plane of its MPI: homography's op sequence (mpi.py:67-81) with torch on CPU."""
    dhw = torch.from_numpy(c["dhw"][c["view2mpi"], -1])
    eye, ray = torch.from_numpy(c["eye"]), torch.from_numpy(c["ray_dir"])
    n, _, h, w = ray.shape
    z_diff = (dhw[:, :1] - eye[:, 2:3]).view(n, 1, 1, 1).expand(n, 1, h, w)
    scale = z_diff / ray[:, 2:3]
    xyz = eye.view(-1, 3, 1, 1) + ray * scale
    return xyz[:, 0].numpy(), xyz[:, 1].numpy()


def base(r8, dhw8, yaws, pitches, seed, align_corners=True):
    ci = cams(r8, IMG, yaws, pitches)
    return dict(rgba_seed=seed, rgba=rand_rgba(seed, (M, N, 4, TEX, TEX)), dhw=np.broadcast_to(dhw8[None, -N:], (M, N, 3)).copy(),
                view2mpi=np.array(VIEW2MPI, np.int32), ray_dir=torch.cat(ci["batch_ray_dir"]).numpy(),
                eye=torch.cat(ci["batch_eye_pos"]).numpy(), z_dir=torch.cat(ci["batch_z_dir"]).numpy(),
                align_corners=np.int32(align_corners))


def copy(c):
    return {k: np.array(v, copy=True) for k, v in c.items()}


def pinned(c, axis, side):
    """(exact, ulp) copies of `c` whose last plane's width (axis "u") or height ("v") puts the extreme pixel on side +1 (max) or
    -1 (min) exactly at u (v) == side, then one ulp beyond.  Returns also the view of that pixel."""
    x, y = last_plane_xy(c)
    t = x if axis == "u" else y
    k = int(np.argmax(side * t))
    ext = np.float32(side * t.flat[k])
    assert ext > 0 and ext >= np.max(-side * t), "the pinned side must be the binding one"
    size = np.float32(2) * ext                                   # exact: u = RN(2x) / (2x) == 1
    col = 2 if axis == "u" else 1
    exact, ulp = copy(c), copy(c)
    exact["dhw"][:, -1, col] = size
    ulp["dhw"][:, -1, col] = np.nextafter(size, np.float32(0))
    return exact, ulp, int(np.unravel_index(k, t.shape)[0])


def main():
    torch.manual_seed(0)
    ref_mpi, ref_r = ref_shim.import_reference()
    r8 = make_renderer(ref_r, 8)
    dhw8 = r8.static_mpi_plane_dhws.numpy()
    cases = {}

    yaws, pitches = [0.2, 0.3, -0.25, 0.15], [0.05, 0.1, -0.05, -0.12]
    clean = base(r8, dhw8, yaws, pitches, 51)
    cases["clean"] = (clean, "ok")

    # the last-plane edges: u and v, max and min side, the extreme pixel in view 0 and in view 2, align_corners True and False
    for tag, ys, ps, ac, axis, side, want_view in (
            ("umax_v0", [-0.3, 0.1, 0.05, 0.2], pitches, True, "u", 1, 0),
            ("umax_v2", [0.05, 0.1, -0.3, 0.2], pitches, True, "u", 1, 2),
            ("umin_v0", [0.3, -0.1, -0.05, -0.2], pitches, True, "u", -1, 0),
            ("vmax_v2", yaws, [0.02, 0.05, 0.15, -0.03], True, "v", 1, 2),
            ("vmin_v0", yaws, [-0.15, 0.0, 0.05, 0.03], True, "v", -1, 0),
            ("umax_acfalse", [0.05, 0.1, -0.3, 0.2], pitches, False, "u", 1, 2),
            ("vmin_acfalse", yaws, [-0.15, 0.0, 0.05, 0.03], False, "v", -1, 0)):
        exact, ulp, view = pinned(base(r8, dhw8, ys, ps, 52, ac), axis, side)
        assert view == want_view, (tag, view)
        cases[tag + "_exact"] = (exact, "ok")
        cases[tag + "_ulp"] = (ulp, "out-of-plane")

    c = copy(clean)                                              # ray_z == 0 and ray_x == ray_y == 0: u = v = NaN on the last plane
    c["ray_dir"][1, :, 9, 4] = 0.0
    cases["nan_ray"] = (c, "out-of-plane")

    eye0_z = clean["eye"][0, 2]
    assert eye0_z > 0 and clean["eye"][1, 2] > eye0_z
    c = copy(clean)                                              # mpi.py:70 is distance >= z_eye[0]: equality passes
    c["dhw"][0, 0, 0] = eye0_z
    cases["dist_eq_eye0"] = (c, "ok")
    c = copy(clean)
    c["dhw"][2, 1, 0] = np.nextafter(eye0_z, np.float32(0))
    cases["dist_ulp_below_eye0"] = (c, "behind-eye")
    c = copy(clean)                                              # only view 0's eye counts: view 1 (same MPI) sees plane 0 behind it
    c["dhw"][0, 0, 0] = (eye0_z + clean["eye"][1, 2]) / 2
    cases["behind_view1_eye"] = (c, "ok")
    c = copy(clean)                                              # only the MPIs a view renders count: MPI 1 has none
    c["dhw"][1, 0, 0] = -0.5
    cases["behind_eye_viewless_mpi"] = (c, "ok")
    c = copy(clean)
    c["dhw"][0, 2, 0] = np.nan
    cases["nan_distance"] = (c, "behind-eye")

    for tag, val, m, want in (("alpha_1p2m23", np.float32(1 + 2.0 ** -23), 2, "alpha"), ("alpha_neg_zero", np.float32(-0.0), 0, "ok"),
                              ("alpha_neg_denormal", -np.float32(2.0 ** -149), 1, "alpha"), ("alpha_nan", np.float32(np.nan), 2, "alpha")):
        c = copy(clean)
        c["rgba"][m, N - 2, 3, 7, 11] = val
        cases[tag] = (c, want)

    names, verdicts, arrs, pool = [], [], {}, []
    for name, (c, want) in cases.items():
        got = verdict(ref_mpi, c)
        assert got == want, (name, got, want)
        names.append(name)
        verdicts.append(got)
        seed = int(c.pop("rgba_seed"))
        rgba = c.pop("rgba")
        patch = np.argwhere(rgba.view(np.int32) != rand_rgba(seed, rgba.shape).view(np.int32))
        assert len(patch) <= 1
        arrs[f"{name}__rgba"] = np.array([seed] + [int(i) for i in patch[0]] if len(patch) else [seed], np.int64)
        arrs[f"{name}__rgba_shape"] = np.array(rgba.shape, np.int64)
        if len(patch):
            arrs[f"{name}__rgba_value"] = rgba[tuple(patch[0])]
        for k, v in c.items():                                   # the other arrays are shared between cases: stored once
            i = next((j for j, p in enumerate(pool) if p.dtype == v.dtype and p.shape == v.shape and p.tobytes() == v.tobytes()), None)
            if i is None:
                i = len(pool)
                pool.append(v)
            arrs[f"{name}__{k}"] = np.int64(i)
        print(f"{name}: {got}")
    arrs.update({f"pool_{j}": p for j, p in enumerate(pool)})
    fixtures = ["nonsquare", "tiny_2mpi_3view_acfalse"]       # verdicts only: their inputs are in their own fixtures
    fixture_verdicts = []
    for name in fixtures:
        z = np.load(os.path.join(OUT, name + ".npz"))
        fixture_verdicts.append(verdict(ref_mpi, {k: z[k] for k in ("rgba", "dhw", "view2mpi", "ray_dir", "eye", "z_dir", "align_corners")}))
        print(f"{name}: {fixture_verdicts[-1]}")
    save("flags_edges", names=np.array(names), verdicts=np.array(verdicts), fixtures=np.array(fixtures),
         fixture_verdicts=np.array(fixture_verdicts), **arrs)


if __name__ == "__main__":
    main()
