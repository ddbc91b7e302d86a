"""Generate tests/golden/envelopes.npz by running the UNMODIFIED reference at the edges of the pose envelopes it trains on
(build container only).

    python oracle/make_golden_envelopes.py      # needs /root/reference; writes tests/golden/envelopes.npz

The reference samples training poses from a truncated Gaussian, mean +- n_truncated_stds x std in yaw and pitch, and sizes its
plane table so that the corners of that envelope just reach the last plane's edge (mpi_utils.py:652-917).  Besides FFHQ
(make_golden.py) it ships two more cameras (curriculums.py:135-204, configs/gmpi.yml:98-110):

    AFHQCat   fov 13.39, planes 2.55-2.8,  sphere r 2.7, yaw / pitch std 0.19 / 0.15, 3 sigma
    MetFaces  fov 12.6,  planes 0.95-1.12, sphere r 1.0, yaw / pitch std 0.339 / 0.133, 2 sigma

Per geometry (keys prefixed "ffhq_", "afhqcat_", "metfaces_"):
  * n8, n32, n96: MPIRenderer.static_mpi_plane_dhws at 8, 32 and 96 planes (AFHQCat and MetFaces; FFHQ's are in ffhq_dhw.npz);
  * yaws, pitches [9]: synth.envelope_poses' order (four corners, four edge midpoints, centre) at scale 1, and yaws_102 /
    pitches_102 at 1.02 x the envelope; c2w, ray_dir, eye, z_dir of MPIRenderer.sample_cam_poses at 20^2 for both (suffix _102);
  * render_img, render_depth, render_c2w, render_angles: MPIRenderer.render (mpi_renderer.py:387-469) of four seeded
    32-plane 128^2 MPIs, one per corner pose, at 64^2 pixels, with the last-plane assert on.  The MPIs are not stored:
    render_rgba_seed / render_rgba_shape regenerate them bit-identically with numpy (conftest.load_golden's rgba_seed).

TEST INFRASTRUCTURE ONLY.
"""
import io
import os
import sys
import zipfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
import ref_shim  # noqa: E402
from make_golden import OUT, cams, make_renderer, quiet, rand_rgba  # noqa: E402
from ml_gmpi_b200 import synth  # noqa: E402
from ml_gmpi_b200.geometry import AFHQCAT, FFHQ, METFACES  # noqa: E402

RENDER_PLANES, RENDER_TEX, RENDER_IMG, CAM_IMG = 32, 128, 64, 20


def reference_kwargs(geo):
    """MPIRenderer keywords of a geometry dict (train.py:277-298 with the dataset's curriculum and FOR_<dataset> block)."""
    kw = dict(ref_shim.FFHQ_KWARGS)
    kw.update(plane_min_d=geo["plane_min_d"], plane_max_d=geo["plane_max_d"], plan_spatial_enlarge_factor=geo["enlarge_factor"],
              plane_distances_sample_method=geo["distance_method"], cam_fov=geo["fov_deg"], sphere_center_z=geo["sphere_center"][2],
              sphere_r=geo["sphere_r"], horizontal_mean=geo["h_mean"], horizontal_std=geo["h_std"], vertical_mean=geo["v_mean"],
              vertical_std=geo["v_std"], cam_pose_n_truncated_stds=geo["n_truncated_stds"], use_confined_volume=geo["confined"])
    return kw


def geometry_arrays(ref_r, tag, geo, seed, tables):
    kw = reference_kwargs(geo)
    out = {}
    if tables:
        for n in (8, 32, 96):
            out[f"n{n}"] = make_renderer(ref_r, n, **kw).static_mpi_plane_dhws.numpy()
    r = make_renderer(ref_r, RENDER_PLANES, **kw)
    for scale, sfx in ((1.0, ""), (1.02, "_102")):
        yaws, pitches = synth.envelope_poses(geo, scale)
        ci = cams(r, CAM_IMG, yaws.tolist(), pitches.tolist())
        out.update({"yaws" + sfx: yaws, "pitches" + sfx: pitches, "c2w" + sfx: ci["batch_tf_c2w"].numpy(),
                    "ray_dir" + sfx: torch.cat(ci["batch_ray_dir"]).numpy(), "eye" + sfx: torch.cat(ci["batch_eye_pos"]).numpy(),
                    "z_dir" + sfx: torch.cat(ci["batch_z_dir"]).numpy()})
    yaws, pitches = synth.envelope_poses(geo)
    shape = (4, RENDER_PLANES, 4, RENDER_TEX, RENDER_TEX)
    rgba = rand_rgba(seed, shape)
    with quiet(), torch.no_grad():
        img, dep, c2w, ang = r.render(torch.from_numpy(rgba), RENDER_IMG, RENDER_IMG, given_yaws=torch.from_numpy(yaws[:4]).view(-1, 1),
                                      given_pitches=torch.from_numpy(pitches[:4]).view(-1, 1), assert_not_out_of_last_plane=True)
    out.update(render_img=img.numpy(), render_depth=dep.numpy(), render_c2w=c2w.numpy(), render_angles=ang.numpy(),
               render_dhw=r.static_mpi_plane_dhws.numpy(), render_rgba_seed=np.int64(seed), render_rgba_shape=np.array(shape))
    return {f"{tag}_{k}": v for k, v in out.items()}


def main():
    torch.manual_seed(0)
    torch.set_num_threads(8)
    _, ref_r = ref_shim.import_reference()
    arrs = {}
    for tag, geo, seed, tables in (("ffhq", FFHQ, 4101, False), ("afhqcat", AFHQCAT, 4102, True), ("metfaces", METFACES, 4103, True)):
        arrs.update(geometry_arrays(ref_r, tag, geo, seed, tables))
    os.makedirs(OUT, exist_ok=True)
    path = os.path.join(OUT, "envelopes.npz")
    # np.savez_compressed stamps the zip members with the current time: a fixed date instead, so that a rerun gives the same bytes
    with zipfile.ZipFile(path, "w", compression=zipfile.ZIP_DEFLATED) as zf:
        for k in sorted(arrs):
            buf = io.BytesIO()
            np.lib.format.write_array(buf, np.asanyarray(arrs[k]), allow_pickle=False)
            info = zipfile.ZipInfo(k + ".npy", date_time=(1980, 1, 1, 0, 0, 0))
            info.compress_type = zipfile.ZIP_DEFLATED
            zf.writestr(info, buf.getvalue())
    print(f"envelopes: {os.path.getsize(path) / 1024:.0f} KiB")


if __name__ == "__main__":
    main()
