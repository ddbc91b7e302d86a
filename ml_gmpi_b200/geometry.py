"""One-off plane geometry of an MPI: plane distances and metric plane sizes (the `dhw` table).

Mirrors (SURVEY.md row A10): sample_distance gmpi/utils/mpi_utils.py:21-53,
compute_plane_dhws_given_cam_pose_spatial_range[_confined] :652-917 and
MPIRenderer.compute_mpi_spatial_volume gmpi/core/mpi_renderer.py:105-152.  The reference walks 10 001
poses in a Python loop (7.7 s); here the pose envelope is evaluated in one vectorised batch (~10 ms).
"""
import numpy as np
import torch

from .camera import PinholeCamera, sphere_poses


def sample_distance(dmin: float, dmax: float, n: int, method: str = "inverse") -> np.ndarray:
    assert 0 < dmin <= dmax and 1 <= n < 9999
    if method == "uniform":
        d = np.linspace(dmin, dmax, n)
    elif method == "log-uniform":
        d = np.exp(np.linspace(np.log(dmin), np.log(dmax), n))
    elif method == "sqrt":
        d = np.linspace(dmin ** 0.5, dmax ** 0.5, n) ** 2
    elif method == "squared":
        d = np.sqrt(np.linspace(dmin ** 2, dmax ** 2, n))
    elif method == "inverse":                                   # uniform in disparity, near -> far
        d = (1.0 / np.linspace(1.0 / dmax, 1.0 / dmin, n))[::-1]
    else:
        raise ValueError(method)
    return np.asarray(d, dtype=np.float32)


def plane_dhw_table(*, n_planes, plane_min_d, plane_max_d, enlarge_factor, distance_method, fov_deg, sphere_center,
                    sphere_r, h_mean, h_std, v_mean, v_std, n_truncated_stds, confined=True, grid=100) -> np.ndarray:
    """-> [n_planes, 3] fp32 (distance, metric height, metric width), planes near -> far."""
    ds = np.clip(sample_distance(plane_min_d, plane_max_d, n_planes, distance_method), plane_min_d, plane_max_d).astype(np.float32)
    far = np.float32(ds[-1])
    h0, h1 = h_mean - n_truncated_stds * h_std, h_mean + n_truncated_stds * h_std
    v0, v1 = v_mean - n_truncated_stds * v_std, v_mean + n_truncated_stds * v_std
    yy, pp = np.meshgrid(np.linspace(h0, h1, grid), np.linspace(v0, v1, grid), indexing="ij")
    yaws = np.concatenate([yy.reshape(-1), [(h0 + h1) / 2]])        # the mid pose is appended last (mpi_utils.py:833)
    pitches = np.concatenate([pp.reshape(-1), [(v0 + v1) / 2]])
    c2w = sphere_poses(torch.from_numpy(yaws), torch.from_numpy(pitches), sphere_center, sphere_r).numpy().astype(np.float64)
    cam = PinholeCamera.from_fov(fov_deg, 4, 4)                      # only ray directions matter (mpi_renderer.py:128)
    rays = np.matmul(c2w[:, :3, :3], cam.border_dirs64()).astype(np.float32)          # [P,3,4]
    eye = c2w[:, :3, 3].astype(np.float32)
    t = (far - eye[:, 2:3]) / rays[:, 2]                                               # mpi_utils.py:632-636
    x = eye[:, 0:1] + rays[:, 0] * t
    y = eye[:, 1:2] + rays[:, 1] * t
    bound = max(np.abs(x).max(), np.abs(y).max())
    assert bound <= 5.0, (f"You have MPI's plane whose boundary value is up to {bound}. This usually means the camera "
                          f"poses's range is too big, which will cause problems for MPI representation.")   # mpi_utils.py:888-894
    mid_h = 2 * np.abs(y[-1]).max()
    mid_w = 2 * np.abs(x[-1]).max()
    rows = []
    for d in ds[:-1]:
        s = 1.0 if confined else float(d) / float(far)                                 # mpi_utils.py:775-779 vs :904-907
        rows.append([d, mid_h * s, mid_w * s])
    rows.append([far, 2 * np.abs(y).max() * enlarge_factor, 2 * np.abs(x).max() * enlarge_factor])
    return np.asarray(rows, dtype=np.float32)


FFHQ = dict(  # curriculums.py:109-116, configs/gmpi.yml:74-96
    plane_min_d=0.95, plane_max_d=1.12, enlarge_factor=1.001, distance_method="inverse", fov_deg=12.6,
    sphere_center=(0.0, 0.0, 1.0), sphere_r=1.0, h_mean=0.0, h_std=0.289, v_mean=0.0, v_std=0.127, n_truncated_stds=2,
    confined=True,
)

AFHQCAT = dict(  # curriculums.py:147-154 (fov, ray_start / ray_end, h_stddev / v_stddev), configs/gmpi.yml:98-103 (FOR_AFHQCat)
    plane_min_d=2.55, plane_max_d=2.8, enlarge_factor=1.001, distance_method="inverse", fov_deg=13.39,
    sphere_center=(0.0, 0.0, 2.7), sphere_r=2.7, h_mean=0.0, h_std=0.19, v_mean=0.0, v_std=0.15, n_truncated_stds=3,
    confined=True,
)

METFACES = dict(  # curriculums.py:185-192, configs/gmpi.yml:105-110 (FOR_MetFaces)
    plane_min_d=0.95, plane_max_d=1.12, enlarge_factor=1.001, distance_method="inverse", fov_deg=12.6,
    sphere_center=(0.0, 0.0, 1.0), sphere_r=1.0, h_mean=0.0, h_std=0.339, v_mean=0.0, v_std=0.133, n_truncated_stds=2,
    confined=True,
)


# ---- texel positions of the planes: what the generator is conditioned on and what LightRenderer shades with --------------------
# Mirrors MPIRenderer.comput_tex_pixels_3d_coords / comput_tex_pixels_3d_normalized_coords_mpi / get_xyz_single_res(only_z) /
# get_xyz_interpolate_ws (gmpi/core/mpi_renderer.py:182-318).  Callers: train.py:328,467,818, fid_evaluation.py:90,
# eval/vis/render_video.py:193-205, eval/prepare_fake_data.py:141-153 -- `mpi_tex_pix_xyz` is also LightRenderer.render's third
# argument (train.py:540,708).  World frame: +X right, +Y down, +Z forward; texel (row r, col c) of plane i sits at
# (lin_w[c]*w_i/2, lin_h[r]*h_i/2, d_i), border texels ON the plane's edge (= align_corners=True sampling).

def texel_xyzd(dhw: torch.Tensor, tex_h: int, tex_w: int) -> torch.Tensor:
    """dhw [N,3] (distance, metric height, metric width) -> [N,tex_h,tex_w,4] = (x, y, z, |xyz|), same dtype/device as dhw.
    (mpi_renderer.py:252-291; the 4th channel is the distance to the world origin, computed before any transformation.)"""
    n = dhw.shape[0]
    half_w = dhw[:, 2:3] / 2.0                                                      # [N,1]
    half_h = dhw[:, 1:2] / 2.0
    x = (torch.linspace(-1, 1, tex_w, device=dhw.device) * half_w).view(n, 1, tex_w)
    y = (torch.linspace(-1, 1, tex_h, device=dhw.device) * half_h).view(n, tex_h, 1)
    out = torch.empty((n, tex_h, tex_w, 4), dtype=dhw.dtype, device=dhw.device)
    out[..., 0] = x
    out[..., 1] = y
    out[..., 2] = dhw[:, 0].view(n, 1, 1)
    out[..., 3] = torch.linalg.vector_norm(out[..., :3], ord=2, dim=3)
    return out


def normalize_xyz(xyz: torch.Tensor, last_plane_hw, plane_min_d: float, plane_max_d: float, xyz_range: str = "-11") -> torch.Tensor:
    """[...,3] world positions -> the MPI volume's unit box: x by the LAST (largest) plane's width, y by its height, z by
    [plane_min_d, plane_max_d]; "01" -> [0,1], "-11" -> [-1,1] (mpi_renderer.py:293-318)."""
    assert xyz_range in ("01", "-11"), xyz_range
    h, w = float(last_plane_hw[0]), float(last_plane_hw[1])
    lo = torch.tensor([-np.float32(w) / 2, -np.float32(h) / 2, plane_min_d], dtype=torch.float32, device=xyz.device)
    hi = torch.tensor([np.float32(w) / 2, np.float32(h) / 2, plane_max_d], dtype=torch.float32, device=xyz.device)
    u = (xyz[..., :3] - lo) / (hi - lo)
    return 2 * u - 1 if xyz_range == "-11" else u


def plane_z(dhw: torch.Tensor, plane_min_d: float, plane_max_d: float, xyz_range: str = "-11"):
    """only_z conditioning: (z [N,1,1,1], z normalised by the depth range) (mpi_renderer.py:183-196)."""
    assert xyz_range in ("01", "-11"), xyz_range
    z = dhw[:, 0].reshape(-1, 1, 1, 1)
    u = (z - plane_min_d) / (plane_max_d - plane_min_d)
    return z, (2 * u - 1 if xyz_range == "-11" else u)


def plane_interpolation_weights(plane_min_d: float, plane_max_d: float, n_src: int, n_tgt: int, method: str = "inverse") -> torch.Tensor:
    """[n_tgt, n_src+2] fp32: row t holds the two linear-interpolation weights of target plane t between its neighbouring
    source planes; columns 0 and n_src+1 are placeholder planes at -/+999999 (mpi_renderer.py:209-250; used to render an MPI
    generated with n_src planes at n_tgt planes, eval/vis/render_video.py:193, eval/prepare_fake_data.py:141).  One
    searchsorted instead of the reference's n_tgt x n_src Python loop."""
    src = torch.empty(n_src + 2, dtype=torch.float32)
    src[0], src[-1] = -999999, 999999
    src[1:-1] = torch.from_numpy(sample_distance(plane_min_d, plane_max_d, n_src, method))
    tgt = torch.from_numpy(sample_distance(plane_min_d, plane_max_d, n_tgt, method))
    j = torch.searchsorted(src, tgt, right=True) - 1                               # src[j] <= tgt < src[j+1]
    lo, hi = src[j], src[j + 1]
    den = (hi - lo) + 1e-8
    ws = torch.zeros((n_tgt, n_src + 2), dtype=torch.float32)
    rows = torch.arange(n_tgt)
    ws[rows, j] = (hi - tgt) / den
    ws[rows, j + 1] = (tgt - lo) / den
    return ws
