"""The arithmetic tests/test_gpu_large_offsets.py rests on, checked without a GPU, so that a later edit to one of its shapes cannot
quietly move a case back below 2^31 elements:
  boundary   which MPI planes, transmittance slabs and frames of each far buffer lie past 2^31 elements (2^32 bytes for the batch)
  census     the stages that read those planes take the staged forward's fast body at every box class 56..88, and its generic body
  plan       each case's descriptor gets the staged kernel at the automatic choice, and the direct one, for its reason, when forced
  memory     each GPU test's declared peak of device bytes fits 24 GiB"""
import numpy as np
import pytest

import mpi_oracle
from ml_gmpi_b200 import _lib
from testlib import (BIG_IMG, BIG_M, BIG_M_FACTORED, BIG_MPI, BIG_N, BIG_PEAK_BYTES, BIG_R, BIG_SLABS, BIG_SLACK, BIG_V_COLOR,
                     BIG_V_GATHER, SMALL_MPI, big_views, forced_kernel, lib)

B31 = 1 << 31


def _first_past(unit, per_slot, slot):
    """The first of the `per_slot` units (of `unit` elements each) of slot `slot` that starts at or past element 2^31."""
    start = slot * per_slot * unit
    return max(0, -(-(B31 - start) // unit))


def test_expanded_mpi_5_holds_planes_32_to_95_past_2_31():
    assert (BIG_M - 1) * BIG_MPI == 2_013_265_920 < B31 < BIG_M * BIG_MPI
    assert _first_past(4 * BIG_IMG, BIG_N, BIG_M - 1) == 32
    assert BIG_M * BIG_MPI == 2_415_919_104                  # 9.7 GB in fp32, 4.8 in fp16, 2.4 in uint8


def test_factored_alpha_and_saved_transmittance_of_slot_21_hold_planes_32_to_95_past_2_31():
    # alpha [22, 96, 1, 1024^2] and the transmittance [22 views, 96, 1024^2] have the same layout: one 1024^2 slab per plane
    assert (BIG_M_FACTORED - 1) * BIG_SLABS == 2_113_929_216 < B31 < BIG_M_FACTORED * BIG_SLABS
    assert _first_past(BIG_IMG, BIG_N, BIG_M_FACTORED - 1) == 32


def test_the_batch_of_four_puts_mpi_2_past_2_31_bytes_and_mpi_3_past_2_32():
    mpi_bytes = BIG_MPI * 4
    assert mpi_bytes == 1_610_612_736
    assert 2 * mpi_bytes > B31 and 3 * mpi_bytes > 1 << 32      # MPI 2 starts at 3.2 GB, MPI 3 at 4.83 GB


def test_output_frames_past_2_31():
    # colour [684, 3, 1024^2]: view 683 starts past 2^31 (view 682's blue channel starts at it); uint8 video [684, 1024^2, 3] alike
    assert (BIG_V_COLOR - 1) * 3 * BIG_IMG > B31 > (BIG_V_COLOR - 2) * 3 * BIG_IMG
    assert (BIG_V_COLOR - 2) * 3 * BIG_IMG + 2 * BIG_IMG == B31
    # fused-gather frames [513, 4, 1024^2]: frame 512 starts at 2^31
    assert (BIG_V_GATHER - 1) * 4 * BIG_IMG == B31


@pytest.mark.parametrize("side", [BIG_R, BIG_R - 1])
def test_range_check_plants_a_colour_at_2_31_and_alpha_last(side):
    """The range tests plant an out-of-range colour value at element 2^31 and an alpha value at the last element; 1023^2 slabs are
    not a whole number of 16-byte loads in fp32 or fp16 (the scalar loops), 1024^2 ones are."""
    slab = side * side
    n = BIG_M * BIG_N * 4 * slab
    assert n > B31
    assert (B31 // slab) % 4 != 3 and ((n - 1) // slab) % 4 == 3
    assert (slab % 4 == 0 and slab % 8 == 0) == (side == BIG_R)


def test_census_of_the_stages_past_2_31():
    """The far views of the expanded and factored tests read planes 32..95 past 2^31: from the pinhole view the forward's stages take
    its fast body at every width class 56..88; every stage of the shuffled view takes the generic body (mode 2), in the forward and
    in the box backward, whose far calls render both views."""
    v = big_views()
    f = mpi_oracle.footprints(v["view2mpi"], v["dhw"], v["ray_dir"], v["eye"], BIG_R, BIG_R, v["ac"])
    past = slice(32, None)
    pin_mode, pin_cls = f["mode"][0][..., past], f["cls"][0][..., past]
    assert all(((pin_mode == 0) & (pin_cls == k)).any() for k in range(56, 96, 8)), np.unique(pin_cls)
    assert (f["mode"][1][..., past] == 2).all()
    # the backward's box (24-row tiles): the pinhole view's far stages take its fast body, the shuffled view's its generic body
    b = mpi_oracle.footprints(v["view2mpi"], v["dhw"], v["ray_dir"], v["eye"], BIG_R, BIG_R, v["ac"], tile=mpi_oracle.BWD_TILE)
    assert (b["mode"][0][..., past] == 0).any() and (b["mode"][1][..., past] == 2).all()
    # the views are two of one MPI: the shuffled view is the pinhole view's rays, permuted
    assert np.array_equal(np.sort(v["ray_dir"][0].reshape(3, -1), 1), np.sort(v["ray_dir"][1].reshape(3, -1), 1))


_A = 1 << 12      # a 16-byte aligned fake address: the plan reads pointers' alignment, never what they point to
PLAN_CASES = {    # name: descriptor fields of each GPU case's far call (NULL pointers count as aligned)
    "expanded-fp32": dict(M=BIG_M, V=2, options=0),
    "expanded-fp16": dict(M=BIG_M, V=2, options=_lib.OPT_MPI_F16),
    "expanded-uint8": dict(M=BIG_M, V=2, options=_lib.OPT_MPI_U8),
    "expanded-backward": dict(M=BIG_M, V=1, options=0),
    "factored": dict(M=BIG_M_FACTORED, V=1, options=0, rgb=_A, alpha=_A, bg_rgb=_A),
    "factored-fp16": dict(M=BIG_M_FACTORED, V=1, options=_lib.OPT_MPI_F16, rgb=_A, alpha=_A, bg_rgb=_A),
    "saved-transmittance": dict(M=1, V=BIG_M_FACTORED, options=0),
    "outputs-color": dict(M=1, V=BIG_V_COLOR, N=SMALL_MPI["N"], Ht=SMALL_MPI["R"], Wt=SMALL_MPI["R"], options=0),
    "outputs-gather": dict(M=1, V=BIG_V_GATHER, N=SMALL_MPI["N"], Ht=SMALL_MPI["R"], Wt=SMALL_MPI["R"], options=0),
    "host-uint8-slot": dict(M=1, V=1, options=_lib.OPT_MPI_U8),
    "batch-of-four": dict(M=4, V=4, options=0),
}


@pytest.mark.parametrize("name", list(PLAN_CASES))
def test_plan_of_each_case(name, lib):
    """Staged at the automatic choice; the direct kernel, and only because it is forced, under the "direct" kernel of the tests."""
    fields = {**dict(N=BIG_N, Ht=BIG_R, Wt=BIG_R, H=BIG_R, W=BIG_R), **PLAN_CASES[name]}
    assert _lib.fwd_plan(_lib.make_desc(**fields)) == (_lib.PLAN_STAGED, 0)
    with forced_kernel("direct"):
        assert _lib.fwd_plan(_lib.make_desc(**fields)) == (_lib.PLAN_DIRECT, 16)      # GMPI_WHY_FORCED


def test_declared_device_peaks_fit_24_gib():
    """Each GPU test's peak (its buffers, plus BIG_SLACK for views, rays and small outputs) fits 24 GiB, so it runs beside other work
    on an 80 GB card; the far buffers themselves pass 2^31 elements."""
    gib = 1 << 30
    table = {k: round((v + BIG_SLACK) / gib, 2) for k, v in BIG_PEAK_BYTES.items()}
    assert all(v <= 24 for v in table.values()), table
    assert BIG_PEAK_BYTES["expanded_backward"] >= 2 * BIG_M * BIG_MPI * 4           # rgba and g_rgba, 9.7 GB each
    assert BIG_PEAK_BYTES["factored"] >= 2 * BIG_M_FACTORED * BIG_SLABS * 4          # alpha and g_alpha, 8.9 GB each
    assert BIG_PEAK_BYTES["saved_transmittance"] >= BIG_M_FACTORED * BIG_SLABS * 4 + BIG_MPI * 8
