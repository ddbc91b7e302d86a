"""CPU checks of the opt-in early ray termination (GMPI_EARLY_STOP): the oracle's per-pixel rule and its error bound, the C ABI's
descriptor sizes and refusals, and the Python plumbing.  The kernels are checked on the GPU in tests/test_gpu_early_stop.py."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

import ml_gmpi_b200 as g
import torch_port
from ml_gmpi_b200 import _lib, service
from conftest import MPI_CASES, ROOT, load_golden
from testlib import lib, max_plane_depth

EDGE_CASES = ["edge_single_plane", "edge_ragged_zero_views", "edge_acfalse_nonsquare", "edge_odd_sizes"]


def render_views_early_stop(batch_rgba, batch_dhw, batch_ray_dir, batch_eye_pos, batch_z_dir, align_corners=True, early_stop=None):
    """The early-stop oracle: oracle/torch_port.render_views (the reference's op sequence, mpi.py:331-436) with the per-pixel rule
    of GMPI_EARLY_STOP added -- a pixel composites plane i only while the transmittance in front of every plane j <= i has
    |T_j| > tau.  early_stop=None is the port's arithmetic op for op (pinned bitwise below)."""
    m_planes = batch_dhw.shape[1]
    rgba = torch.cat([batch_rgba[k:k + 1].expand(r.shape[0], -1, -1, -1, -1) for k, r in enumerate(batch_ray_dir)], 0)
    dhw = torch.cat([batch_dhw[k:k + 1].expand(r.shape[0], -1, -1) for k, r in enumerate(batch_ray_dir)], 0)
    rays, eyes, zdirs = torch.cat(batch_ray_dir, 0), torch.cat(batch_eye_pos, 0), torch.cat(batch_z_dir, 0)
    nv, _, ih, iw = rays.shape
    th, tw = rgba.shape[-2:]
    rays_f = rays.unsqueeze(1).expand(-1, m_planes, -1, -1, -1).reshape(nv * m_planes, 3, ih, iw)
    eyes_f = eyes.unsqueeze(1).expand(-1, m_planes, -1).reshape(nv * m_planes, 3)
    zdirs_f = zdirs.unsqueeze(1).expand(-1, m_planes, -1).reshape(nv * m_planes, 3)
    rgb, disparity, alpha = torch_port.warp_planes(rgba.reshape(nv * m_planes, 4, th, tw), dhw.reshape(nv * m_planes, 3), eyes_f,
                                                   rays_f, zdirs_f, align_corners)
    z = (1 / disparity).reshape(nv, m_planes, 1, ih, iw)
    alpha = alpha.reshape(nv, m_planes, 1, ih, iw)
    rgb = rgb.reshape(nv, m_planes, 3, ih, iw)
    shifted = torch.cat([torch.ones_like(alpha[:, :1]), 1 - alpha + 1e-10], 1)
    trans = torch.cumprod(shifted, dim=1)[:, :-1]
    wgt = alpha * trans
    if early_stop is not None:
        live = torch.cumprod((~(trans.abs() <= early_stop)).to(trans.dtype), dim=1) > 0
        wgt = torch.where(live, wgt, torch.zeros_like(wgt))
    return torch.sum(wgt * rgb, dim=1), torch.sum(wgt * z, dim=1)


def _groups(gd):
    v2m = gd["view2mpi"]
    idx = [np.nonzero(v2m == m)[0] for m in range(gd["rgba"].shape[0])]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a))
    return (t(gd["rgba"]), t(gd["dhw"]), [t(gd["ray_dir"][i]) for i in idx], [t(gd["eye"][i]) for i in idx],
            [t(gd["z_dir"][i]) for i in idx])


def _port(gd, early_stop=None):
    color, depth = render_views_early_stop(*_groups(gd), align_corners=bool(gd["align_corners"]), early_stop=early_stop)
    return color.numpy(), depth.numpy()


@pytest.mark.parametrize("name", MPI_CASES + EDGE_CASES)
def test_oracle_tau_zero_and_off_are_bitwise_the_torch_port(name):
    """Without tau and at tau = 0 the early-stop oracle is bit for bit oracle/torch_port.render_views (itself bit-identical to
    the reference on these fixtures, tests/test_oracle_golden.py)."""
    gd = load_golden(name)
    c0, d0 = torch_port.render_views(*_groups(gd), align_corners=bool(gd["align_corners"]))
    c0, d0 = c0.numpy(), d0.numpy()
    for tau in (None, 0.0):
        c, d = _port(gd, early_stop=tau)
        assert np.array_equal(c.view(np.uint32), c0.view(np.uint32)) and np.array_equal(d.view(np.uint32), d0.view(np.uint32)), tau


@pytest.mark.parametrize("tau", [2.0 ** -24, 1e-3])
@pytest.mark.parametrize("name", MPI_CASES + EDGE_CASES)
def test_oracle_early_stop_stays_within_its_bound(name, tau):
    """Each colour channel moves by at most tau, depth by at most tau * (the pixel's largest plane depth)."""
    gd = load_golden(name)
    c0, d0 = _port(gd)
    c, d = _port(gd, early_stop=tau)
    slack = 2e-6
    assert np.max(np.abs(c - c0)) <= tau + slack * max(1.0, float(np.max(np.abs(c0))))
    assert np.all(np.abs(d - d0) <= tau * max_plane_depth(gd) * (1 + 1e-5) + slack * float(np.max(np.abs(d0))))


def test_oracle_early_stop_drops_planes_behind_opaque_content():
    """alpha_one_planes has opaque planes: tau = 1e-3 must actually change something, or the bound test checks nothing."""
    gd = load_golden("alpha_one_planes")
    c0, _ = _port(gd)
    c, _ = _port(gd, early_stop=0.05)
    assert np.max(np.abs(c - c0)) > 0.0


def test_header_option_bit_and_descriptor_sizes():
    hdr = open(os.path.join(ROOT, "include", "gmpi_mpi_render.h")).read()
    for name, val in [("GMPI_EARLY_STOP", _lib.OPT_EARLY_STOP), ("GMPI_U8_ROUND_HALF_UP", _lib.OPT_U8_ROUND_HALF_UP)]:
        m = re.search(rf"#define {name} (\d+)u", hdr)
        assert m and int(m.group(1)) == val, name
    assert _lib.RenderDesc._fields_[-1] == ("early_stop", ctypes.c_float)
    # the descriptor before early_stop was appended ends at the stream pointer
    assert _lib.RENDER_DESC_V2_BYTES == _lib.RenderDesc.stream.offset + ctypes.sizeof(ctypes.c_void_p)
    assert ctypes.sizeof(_lib.RenderDesc) > _lib.RENDER_DESC_V2_BYTES


def _desc(p, **kw):
    base = dict(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4, rgba=p, view2mpi=p, dhw=p, ray_dir=p, eye=p, z_dir=p)
    base.update(kw)
    return _lib.make_desc(**base)


def test_descriptor_of_the_previous_size_is_accepted(lib):
    d = _lib.make_desc(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4)
    d.struct_bytes = _lib.RENDER_DESC_V2_BYTES
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"null input" in lib.gmpi_last_error()   # past the size check
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == 1 and b"null input" in lib.gmpi_last_error()
    for bad in (8, _lib.RENDER_DESC_V2_BYTES + 4):
        d.struct_bytes = bad
        assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"struct_bytes" in lib.gmpi_last_error()
    # the old size has no early_stop field: the bit is refused there
    d = _lib.make_desc(M=1, V=1, N=1, Ht=4, Wt=4, H=4, W=4, options=_lib.OPT_EARLY_STOP)
    d.struct_bytes = _lib.RENDER_DESC_V2_BYTES
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"GMPI_EARLY_STOP" in lib.gmpi_last_error()


def test_early_stop_is_refused_for_training_and_backward(lib):
    buf = (ctypes.c_float * 64)()
    p = ctypes.addressof(buf)
    es = _lib.OPT_EARLY_STOP
    d = _desc(p, options=es, early_stop=1e-3, color=p, depth=p, flags=p, transmittance=p)
    assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 3 and b"transmittance" in lib.gmpi_last_error()
    d = _desc(p, options=es, early_stop=1e-3, g_color=p, g_rgba=p, transmittance=p)
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == 3 and b"forward-only" in lib.gmpi_last_error()
    d = _desc(p, options=es, early_stop=1e-3, g_color=p, g_rgba=p)
    assert lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)) == 3
    for bad in (-1e-3, 1.0, float("nan")):
        d = _desc(p, options=es, early_stop=bad, color=p, depth=p, flags=p)
        assert lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)) == 1 and b"early_stop" in lib.gmpi_last_error()
    # the classic entry points have no threshold field
    rc = lib.gmpi_mpi_render_fwd(p, p, p, p, p, p, p, p, p, 1, 1, 1, 4, 4, 4, 4, es, None)
    assert rc == 1 and b"early_stop" in lib.gmpi_last_error()
    rc = lib.gmpi_mpi_render_fwd_train(p, p, p, p, p, p, p, p, p, p, 1, 1, 1, 4, 4, 4, 4, es, None)
    assert rc == 3
    skipped, total = ctypes.c_ulonglong(), ctypes.c_ulonglong()
    assert lib.gmpi_debug_fwd_early_stop_stats(None, ctypes.byref(total)) == 1


def _inputs(requires_grad):
    rgba = torch.rand(1, 2, 4, 8, 8).requires_grad_(requires_grad)
    ray = torch.zeros(1, 3, 4, 4); ray[:, 2] = 1
    return rgba, torch.rand(1, 2, 3), torch.zeros(1, dtype=torch.int32), ray, torch.zeros(1, 3), torch.tensor([[0., 0., 1.]])


def test_early_stop_with_grad_raises_a_clear_error():
    rgba, dhw, v2m, ray, eye, z = _inputs(True)
    with pytest.raises(RuntimeError, match="early_stop is forward-only"):
        g.render_views(rgba, dhw, v2m, ray, eye, z, early_stop=1e-3)
    rgb, alpha = torch.rand(1, 3, 8, 8, requires_grad=True), torch.rand(1, 2, 1, 8, 8)
    with pytest.raises(RuntimeError, match="early_stop is forward-only"):
        g.render_views_factored(rgb, alpha, dhw, v2m, ray, eye, z, early_stop=0.0)
    # without autograd the call gets as far as the device check
    with torch.no_grad(), pytest.raises(RuntimeError, match="CUDA devices only"):
        g.render_views(rgba, dhw, v2m, ray, eye, z, early_stop=1e-3)
    with pytest.raises(RuntimeError, match="CUDA devices only"):
        g.render_views(rgba.detach(), dhw, v2m, ray, eye, z, early_stop=1e-3)
    with pytest.raises(RuntimeError, match="CUDA devices only"):          # early stop off: grad is fine
        g.render_views(rgba, dhw, v2m, ray, eye, z)


def test_render_frames_and_frame_gather_take_early_stop():
    import inspect
    from ml_gmpi_b200.dist import FrameGather
    assert inspect.signature(g.render_frames).parameters["early_stop"].default is None
    assert inspect.signature(FrameGather.render).parameters["early_stop"].default is None


def test_service_drivers_pass_early_stop_through():
    seen = []

    def video(rgba, dhw, c2w, img_size, fov, near, far, fast, factored, **kw):
        seen.append(kw)
        V = c2w.shape[0]
        return torch.zeros(V, img_size, img_size, 3, dtype=torch.uint8), torch.zeros(V, img_size, img_size, 1, dtype=torch.uint8)
    kw = dict(img_size=4, fov_deg=12.0, ray_start=0.9, ray_end=1.1, sphere_center=np.array([0, 0, 1.0]), sphere_r=1.0)
    service.render_video_frames(None, torch.zeros(1, 2, 3), [0.1, 0.2], render_fn=video, **kw)
    service.render_video_frames(None, torch.zeros(1, 2, 3), [0.1, 0.2], render_fn=video, early_stop=2.0 ** -24, **kw)
    assert seen == [{}, {"early_stop": 2.0 ** -24}]

    def fid(renderer, batch, img_size, yaws, pitches, **kw):
        seen.append(kw)
        return torch.zeros(batch.shape[0], img_size, img_size, 3, dtype=torch.uint8)
    service.dump_fid_images(None, lambda k: torch.zeros(2, 1, 4, 2, 2), 2, 0, 1, 4, writer=lambda i, im: None, render_fn=fid,
                            early_stop=1e-3)
    assert seen[-1] == {"early_stop": 1e-3}

    class R:
        horizontal_mean, horizontal_std, vertical_mean, vertical_std = 0.0, 0.3, 0.0, 0.1
        cam_pose_n_truncated_stds, cam_sample_method = 2, "truncated_gaussian"

    def ev(renderer, batch, n_imgs, img_size, yaws, pitches, **kw):
        seen.append(kw)
        V = batch.shape[0] * n_imgs
        return torch.zeros(V, 3, img_size, img_size), torch.ones(V, 1, img_size, img_size)
    service.render_eval_views(R(), torch.zeros(1, 2, 4, 4, 4), n_imgs=2, img_size=4, render_fn=ev, early_stop=0.0)
    assert seen[-1] == {"early_stop": 0.0}
    import inspect
    for fn in (service._default_video_render, service._default_fid_render, service._default_eval_render):
        assert inspect.signature(fn).parameters["early_stop"].default is None


def test_head_workload_is_transparent_with_an_opaque_head():
    from ml_gmpi_b200 import synth
    a = synth.head_alpha(96, 128)
    assert float(a[-1].min()) == 1.0 and float(a[:40].max()) == 0.0
    assert 0.5 <= float(a[:-1].amax(0).mean()) <= 0.7                 # the head covers about 60 % of the frame
    assert set(np.unique(a.numpy()).tolist()) <= {0.0, 1.0}
