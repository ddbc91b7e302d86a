"""Pins the CPU oracle (oracle/mpi_oracle.c, oracle/torch_port.py) to outputs of the unmodified
reference (tests/golden/*.npz, produced by oracle/make_golden.py from /root/reference).

Tolerance: the oracle reproduces the reference's fp32 coordinate arithmetic bit for bit, so the
residual is summation-order noise of well-conditioned sums: <= 2e-6 of max|ref| (the parity bar
for the product is 1e-4, SURVEY.md section 8c)."""
import numpy as np
import pytest
import torch

import mpi_oracle
import torch_port
from conftest import MPI_CASES, load_golden, rel_err
from testlib import FLAG_CASES, FORWARD_FLAGS

TOL = 2e-6
# The range check's flag word for each verdict of the reference (the forward's: testlib.FORWARD_FLAGS).
RANGE_FLAGS = {"ok": 0, "alpha": mpi_oracle.FLAG_ALPHA_RANGE | mpi_oracle.FLAG_RGBA_RANGE, "behind-eye": 0, "out-of-plane": 0}
_fz = load_golden("flags_edges")
FIXTURE_VERDICTS = dict(zip(_fz["fixtures"].tolist(), _fz["fixture_verdicts"].tolist()))


@pytest.mark.parametrize("name", MPI_CASES + ["c1_full_256"])
def test_c_oracle_forward_matches_reference(name):
    g = load_golden(name)
    color, depth, flags = mpi_oracle.forward(g["rgba"], g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], g["z_dir"],
                                             align_corners=bool(g["align_corners"]), check_last_plane=True, nthreads=4)
    assert rel_err(color, g["color"]) <= TOL
    assert rel_err(depth, g["depth"]) <= TOL
    if name == "out_of_plane":
        assert flags & mpi_oracle.FLAG_LAST_PLANE_OOB
    elif name in FIXTURE_VERDICTS:         # the reference's own verdict on the fixture (oracle/make_golden_flags.py)
        assert flags == FORWARD_FLAGS[FIXTURE_VERDICTS[name]], (flags, FIXTURE_VERDICTS[name])
    else:
        assert flags == 0


@pytest.mark.parametrize("name", [n for n in MPI_CASES if n != "c2_small_4x32x64"])
def test_c_oracle_backward_matches_reference_autograd(name):
    g = load_golden(name)
    gr = mpi_oracle.backward(g["rgba"], g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], g["z_dir"], g["g_color"],
                             g.get("g_depth"), align_corners=bool(g["align_corners"]))
    assert rel_err(gr, g["g_rgba"]) <= 5e-6


@pytest.mark.parametrize("name", ["tiny_2mpi_3view", "alpha_one_planes", "out_of_plane", "nonsquare"])
def test_c_oracle_over_composite_matches_old_forward(name):
    """MPI.old_forward (mpi.py:280-304) is the reference's own second formulation."""
    g = load_golden(name)
    c, d = mpi_oracle.forward_over(g["rgba"], g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], g["z_dir"],
                                   align_corners=bool(g["align_corners"]))
    assert rel_err(c, g["color_over"]) <= TOL
    assert rel_err(d, g["depth_over"]) <= TOL
    # and the two formulations agree up to the 1e-10 epsilon (SURVEY.md section 4 (iv))
    assert rel_err(c, g["color"]) <= 1e-5


def _groups(g):
    v2m = g["view2mpi"]
    M = g["rgba"].shape[0]
    ray, eye, z = torch.from_numpy(g["ray_dir"]), torch.from_numpy(g["eye"]), torch.from_numpy(g["z_dir"])
    idx = [np.nonzero(v2m == m)[0] for m in range(M)]
    return [ray[i] for i in idx], [eye[i] for i in idx], [z[i] for i in idx]


@pytest.mark.parametrize("name", MPI_CASES)
def test_torch_port_is_bit_identical_to_reference(name):
    g = load_golden(name)
    rays, eyes, zs = _groups(g)
    rgba = torch.from_numpy(g["rgba"]).clone().requires_grad_(True)
    color, depth = torch_port.render_views(rgba, torch.from_numpy(g["dhw"]), rays, eyes, zs,
                                           align_corners=bool(g["align_corners"]))
    assert np.array_equal(color.detach().numpy(), g["color"])
    assert np.array_equal(depth.detach().numpy(), g["depth"])
    if "g_rgba" in g:
        loss = (color * torch.from_numpy(g["g_color"])).sum()
        if "g_depth" in g:
            loss = loss + (depth * torch.from_numpy(g["g_depth"])).sum()
        loss.backward()
        assert rel_err(rgba.grad.numpy(), g["g_rgba"]) <= 1e-6


def test_coordinate_stage_is_bit_exact_vs_torch_ops():
    """The C oracle's (ix, iy) must equal what torch's elementwise ops + grid_sampler_unnormalize
    produce, bit for bit (SURVEY.md section 7 H1)."""
    g = load_golden("c1_small_64")
    Ht, Wt = g["rgba"].shape[-2:]
    co = mpi_oracle.coords(g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], Ht, Wt, True)
    ray = torch.from_numpy(g["ray_dir"]); eye = torch.from_numpy(g["eye"]); dhw = torch.from_numpy(g["dhw"])
    for i in range(dhw.shape[1]):
        d, h, w = dhw[0, i]
        t = (d - eye[0, 2]) / ray[0, 2]
        x = eye[0, 0] + ray[0, 0] * t
        y = eye[0, 1] + ray[0, 1] * t
        u = 2 * x / w
        v = 2 * y / h
        ix = ((u + 1) / 2) * (Wt - 1)
        iy = ((v + 1) / 2) * (Ht - 1)
        assert np.array_equal(co[0, i, 0], ix.numpy())
        assert np.array_equal(co[0, i, 1], iy.numpy())


def test_oracle_range_flags():
    g = load_golden("tiny_2mpi_3view")
    assert mpi_oracle.check_range(g["rgba"]) == 0
    bad = g["rgba"].copy(); bad[0, 0, 1, 0, 0] = 1.5
    assert mpi_oracle.check_range(bad) == mpi_oracle.FLAG_RGBA_RANGE
    bad = g["rgba"].copy(); bad[1, 2, 3, 3, 3] = -0.1
    assert mpi_oracle.check_range(bad) & mpi_oracle.FLAG_ALPHA_RANGE


# Edge cases of the reference's forward that only the ORACLE is pinned with (oracle/make_golden_edge.py): a single plane, an MPI
# without views between MPIs with views, align_corners=False on a non-square texture, sizes that are multiples of nothing.
EDGE_CASES = ["edge_single_plane", "edge_ragged_zero_views", "edge_acfalse_nonsquare", "edge_odd_sizes"]


@pytest.mark.parametrize("name", EDGE_CASES)
def test_edge_cases_c_oracle_and_torch_port(name):
    g = load_golden(name)
    ac = bool(g["align_corners"])
    color, depth, _ = mpi_oracle.forward(g["rgba"], g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], g["z_dir"],
                                         align_corners=ac, check_last_plane=False, nthreads=2)
    assert color.shape == g["color"].shape and rel_err(color, g["color"]) <= TOL and rel_err(depth, g["depth"]) <= TOL
    gr = mpi_oracle.backward(g["rgba"], g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], g["z_dir"], g["g_color"], g.get("g_depth"),
                             align_corners=ac)
    assert rel_err(gr, g["g_rgba"]) <= 5e-6
    c_over, d_over = mpi_oracle.forward_over(g["rgba"], g["view2mpi"], g["dhw"], g["ray_dir"], g["eye"], g["z_dir"], align_corners=ac)
    assert rel_err(c_over, g["color_over"]) <= TOL and rel_err(d_over, g["depth_over"]) <= TOL
    rays, eyes, zs = _groups(g)
    pc, pd = torch_port.render_views(torch.from_numpy(g["rgba"]), torch.from_numpy(g["dhw"]), rays, eyes, zs, align_corners=ac)
    assert np.array_equal(pc.numpy(), g["color"]) and np.array_equal(pd.numpy(), g["depth"])
    if name == "edge_ragged_zero_views":
        assert g["view2mpi"].tolist() == [0, 0, 2] and not gr[1].any()          # the view-less MPI gets an exactly zero gradient
    if name == "edge_single_plane":                                             # N = 1: colour = alpha_0 * rgb_0 of the warped plane
        assert g["rgba"].shape[1] == 1 and float(np.max(color)) <= 1.0


@pytest.mark.parametrize("name,verdict,case", FLAG_CASES, ids=[n for n, _, _ in FLAG_CASES])
def test_oracle_flags_are_the_reference_verdict(name, verdict, case):
    """Crafted cases at the edges of the reference's three data-dependent checks (oracle/make_golden_flags.py): |u| or |v| exactly
    1 on the last plane and one ulp beyond, a NaN ray, a plane distance equal to view 0's eye z and one ulp below, a plane behind
    a later view's eye, a plane behind the eye in an MPI no view renders, a NaN distance, alpha of 1 + 2^-23, -0.0, -denormal and
    NaN.  The oracle's forward (with and without the last-plane check) and range check give exactly the bit the reference's
    verdict implies, and no other."""
    c = case
    args = (c["rgba"], c["view2mpi"], c["dhw"], c["ray_dir"], c["eye"], c["z_dir"])
    ac = bool(c["align_corners"])
    assert mpi_oracle.forward(*args, align_corners=ac, check_last_plane=True)[2] == FORWARD_FLAGS[verdict]
    assert mpi_oracle.forward(*args, align_corners=ac, check_last_plane=False)[2] == \
        FORWARD_FLAGS[verdict] & ~mpi_oracle.FLAG_LAST_PLANE_OOB
    assert mpi_oracle.check_range(c["rgba"]) == RANGE_FLAGS[verdict]
