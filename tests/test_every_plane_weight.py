"""The equal-weight MPIs of the full-size GPU tests (synth.equal_weight_alpha) put every plane where the parity bar sees it, and the
shapes those tests run cover every box the staged kernels pick.  CPU only: the oracle and its texel coordinates.

With U(0, 1) alpha the transmittance falls as e^-i, so planes past ~25 of a 96-plane render move the colour and the gradient by
less than the bar (max|ours - ref| / max|ref| <= 2e-5): a kernel that mis-sampled them would pass.  Here every plane of the
equal-weight MPI must move the oracle's colour, and own a share of its gradient, by 100 x the bar; the U(0, 1) MPI must not, at
plane 48, which is why the GPU tests need the equal-weight input."""
import functools

import numpy as np
import pytest

import mpi_oracle
from ml_gmpi_b200 import synth
from conftest import rel_err

BAR = 2e-5                 # the GPU parity bar (tests/test_gpu_parity.py EXPECT)
TEETH = 100 * BAR
PLANES = (0, 12, 24, 48, 72, 94, 95)
N, RES = 96, 256


@functools.lru_cache(maxsize=None)
def _problem(alpha):
    c = synth.make_case(n_planes=N, tex=RES, img=RES, n_mpi=1, seed=1234, alpha=alpha, last_alpha_one=True)
    geo = tuple(t.numpy() for t in (c.view2mpi, c.dhw, c.ray_dir, c.eye, c.z_dir))
    return c.rgba.numpy(), geo


def _colour(rgba, geo):
    return mpi_oracle.forward(rgba, *geo, nthreads=8)[0]


def _moved(alpha, k, channels):
    """max |colour change| / max |colour| when plane k's `channels` are rolled by one texel along x."""
    rgba, geo = _problem(alpha)
    rolled = rgba.copy()
    rolled[:, k, channels] = np.roll(rgba[:, k, channels], 1, axis=-1)
    return rel_err(_colour(rolled, geo), _colour(rgba, geo))


@functools.lru_cache(maxsize=None)
def _plane_shares(alpha):
    """Per plane: max |d alpha| and max |d rgb| over the global max |d rgba|, for colour and depth upstream gradients."""
    rgba, geo = _problem(alpha)
    gen = np.random.default_rng(3)
    gc = gen.standard_normal((1, 3, RES, RES)).astype(np.float32)
    gd = gen.standard_normal((1, 1, RES, RES)).astype(np.float32)
    G = np.abs(mpi_oracle.backward(rgba, *geo, gc, gd, nthreads=8))
    top = G.max()
    return G[0, :, 3].max(axis=(-2, -1)) / top, G[0, :, :3].max(axis=(-3, -2, -1)) / top


@pytest.mark.parametrize("k", PLANES)
def test_every_plane_moves_the_colour(k):
    """Plane k's rgb, and its alpha, rolled by one texel: the colour moves by >= 100 x the bar.  (The last plane's alpha is 1 on
    every texel, so rolling it changes nothing: only its rgb is rolled.)"""
    rgb = _moved("equal_weight", k, slice(0, 3))
    a = _moved("equal_weight", k, slice(3, 4)) if k < N - 1 else None
    print(f"plane {k}: rgb rolled {rgb:.3g}, alpha rolled {a}")
    assert rgb >= TEETH and (a is None or a >= TEETH), (rgb, a)


def test_every_plane_owns_a_share_of_the_gradient():
    da, drgb = _plane_shares("equal_weight")
    print("d alpha share, min over planes", float(da.min()), "d rgb share", float(drgb.min()))
    assert (da >= TEETH).all(), np.nonzero(da < TEETH)[0]
    assert (drgb >= TEETH).all(), np.nonzero(drgb < TEETH)[0]


def test_uniform_alpha_hides_plane_48():
    """The same checks on U(0, 1) alpha fail at plane 48: its colour and gradient sit below the bar itself."""
    rgb, a = _moved("uniform", 48, slice(0, 3)), _moved("uniform", 48, slice(3, 4))
    da, drgb = _plane_shares("uniform")
    print(f"uniform plane 48: rgb rolled {rgb:.3g}, alpha rolled {a:.3g}, d alpha {da[48]:.3g}, d rgb {drgb[48]:.3g}")
    assert max(rgb, a, da[48], drgb[48]) < BAR


def test_equal_weight_alpha():
    """min(1, u * 2 / (N - i)) with u ~ U(0, 1) per texel, the last plane 1; the mean compositing weight of every plane ~ 1 / N."""
    import torch
    a = synth.equal_weight_alpha((2, N, 64, 64), torch.Generator().manual_seed(0)).numpy().astype(np.float64)
    assert a.shape == (2, N, 64, 64) and a.min() >= 0 and a.max() <= 1 and (a[:, -1] == 1).all()
    assert len(np.unique(a[:, N // 2])) > 1000                     # varies per texel
    T = np.cumprod(np.concatenate([np.ones_like(a[:, :1]), 1 - a[:, :-1]], 1), 1)
    w = (a * T).mean(axis=(0, 2, 3))
    assert np.allclose(w, 1 / N, rtol=0.25), w
    dflt = synth.make_case(n_planes=8, tex=16, img=16, n_mpi=1, seed=5).rgba
    assert torch.equal(dflt, synth.make_case(n_planes=8, tex=16, img=16, n_mpi=1, seed=5, alpha="uniform").rgba)


# ------------------------------------------------------------------------------------------------------------------------------
# coverage: the producer's box classes at the shapes the GPU tests run on equal-weight data
# ------------------------------------------------------------------------------------------------------------------------------
_C4_YAWS = np.linspace(0.5, -0.5, 120).astype(np.float32)[::8]
# name: (make_case arguments, whether the test runs the box backward too)
SHAPES = {
    "full_32x256_8views": (dict(n_planes=32, tex=256, img=256, n_mpi=8), False),
    "full_96x512_2views": (dict(n_planes=96, tex=512, img=512, n_mpi=2), False),
    "c3_96x1024": (dict(n_planes=96, tex=1024, img=1024, n_mpi=1), True),
    "c5_96x512_4mpis": (dict(n_planes=96, tex=512, img=512, n_mpi=4, seed=99), True),
    "four_views_48x512": (dict(n_planes=48, tex=512, img=512, n_mpi=1, views_per_mpi=4, seed=21), True),
    "c4_video_15views": (dict(n_planes=96, tex=512, img=512, n_mpi=1, views_per_mpi=15, yaws=_C4_YAWS,
                              pitches=np.zeros(15, np.float32)), False),
    "deterministic_4x96x1024": (dict(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=3), True),
}
# where a footprint is too wide or tall for a ring stage (mode 2, the generic body): (forward, backward)
MODE2 = {"full_32x256_8views": (True, True), "full_96x512_2views": (True, True), "four_views_48x512": (False, True),
         "deterministic_4x96x1024": (True, True)}


def _footprints(kw, **extra):
    c = synth.make_case(rgba=False, **kw)
    return mpi_oracle.footprints(c.view2mpi.numpy(), c.dhw.numpy(), c.ray_dir.numpy(), c.eye.numpy(), kw["tex"], kw["tex"], **extra)


@pytest.mark.parametrize("name", list(SHAPES))
def test_every_box_class_occurs(name):
    kw, backward = SHAPES[name]
    for tile, check in ((mpi_oracle.FWD_TILE, True), (mpi_oracle.BWD_TILE, backward)):
        if not check:
            continue
        f = _footprints(kw, tile=tile)
        counts = {k: int((f["cls"] == k).sum()) for k in range(56, 96, 8)}
        print(name, tile, counts, "mode 2:", int((f["mode"] == 2).sum()))
        assert all(v > 0 for v in counts.values()), (tile, counts)
        assert bool((f["mode"] == 2).any()) == MODE2.get(name, (False, False))[tile == mpi_oracle.BWD_TILE], tile
        # class 88 (kMaxBW) behind plane 25, where U(0, 1) alpha would leave it unseen
        assert (f["cls"][..., 25:] == 88).any()


@pytest.mark.parametrize("kw", [dict(n_planes=96, tex=1024, img=1024, n_mpi=1, seed=1234),
                                dict(n_planes=48, tex=512, img=512, n_mpi=1, views_per_mpi=4, seed=21)],
                         ids=["bench_96x1024", "views4_48x512"])
def test_the_factored_forward_boxes_occur(kw):
    f = _footprints(kw, wide=True)
    assert (f["cls"] == 64).any() and (f["cls"] == 96).any()


def test_footprints_match_the_producer_arithmetic_on_a_hand_case():
    """One tile whose corner coordinates are known: an identity-like view of a 256^2 texture at 256^2 pixels sees, on each plane, a
    box about one tile wide; the helper's fields follow the producer's formulas from those corners."""
    kw = dict(n_planes=4, tex=256, img=256, n_mpi=1, seed=1, yaws=[0.0], pitches=[0.0])
    c = synth.make_case(rgba=False, **kw)
    f = mpi_oracle.footprints(c.view2mpi.numpy(), c.dhw.numpy(), c.ray_dir.numpy(), c.eye.numpy(), 256, 256)
    co = mpi_oracle.coords(c.view2mpi.numpy(), c.dhw.numpy(), c.ray_dir.numpy(), c.eye.numpy(), 256, 256)
    ty, tx = 2, 1                                             # pixels 60..89 x 64..127
    fx = np.floor(co[0, :, 0][:, [60, 60, 89, 89], [64, 127, 64, 127]]).astype(np.int64)
    fy = np.floor(co[0, :, 1][:, [60, 60, 89, 89], [64, 127, 64, 127]]).astype(np.int64)
    bx0 = (fx.min(1) - 1) // 4 * 4
    assert np.array_equal(f["bx0"][0, ty, tx], bx0)
    assert np.array_equal(f["need_w"][0, ty, tx], fx.max(1) - bx0 + 3)
    assert np.array_equal(f["need_h"][0, ty, tx], fy.max(1) - fy.min(1) + 4)
    assert (f["mode"][0, ty, tx] == 0).all()
    assert np.array_equal(f["cls"][0, ty, tx], 56 + 8 * np.maximum(0, -(-(f["need_w"][0, ty, tx] - 56) // 8)))
