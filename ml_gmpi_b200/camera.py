"""Pinhole camera rays and sphere-orbit poses: the small per-view inputs of the render path.

Mirrors (SURVEY.md section 8a rows A2-A4), re-derived rather than transcribed:
  Camera / gen_cam            gmpi/core/camera.py:13-211, gmpi/utils/cam_utils.py:16-22
  gen_sphere_path + helpers   gmpi/utils/cam_utils.py:481-622,687-821
  MPIRenderer.sample_cam_poses / view_info_from_c2w_mat   gmpi/core/mpi_renderer.py:320-385

Conventions (reference): world/MPI frame +X right, +Y down, +Z forward; the camera sits on a sphere
(centre `sphere_center`, radius r) and looks at the centre; yaw moves it horizontally, pitch
vertically; pixel centres at (+0.5, +0.5); principal point (w/2, h/2); f = w / (2 tan(fov/2)).
"""
import math
from typing import Optional, Tuple

import numpy as np
import torch


def focal_from_fov(fov_deg: float, width: int) -> float:
    return width / (2.0 * math.tan(math.pi * fov_deg / 360.0))          # mpi_renderer.py:88-89


class PinholeCamera:
    """Per-pixel unit rays in camera space (fp64 -> fp32, cached), rotated to world space per view."""

    def __init__(self, height: int, width: int, focal: float, ray_from_pix_center: bool = True):
        self.height, self.width, self.focal = int(height), int(width), float(focal)
        self.ray_from_pix_center = ray_from_pix_center
        self._rays = {}

    @classmethod
    def from_fov(cls, fov_deg: float, height: int, width: int):
        return cls(height, width, focal_from_fov(fov_deg, width))

    def _cam_dirs64(self) -> np.ndarray:
        off = 0.5 if self.ray_from_pix_center else 0.0                   # camera.py:63-66
        xs = (np.arange(self.width, dtype=np.float64) + off - self.width / 2.0) / self.focal
        ys = (np.arange(self.height, dtype=np.float64) + off - self.height / 2.0) / self.focal
        d = np.stack(np.broadcast_arrays(xs[None, :], ys[:, None], np.ones((1, 1))), 0)     # K^-1 [u v 1]
        return (d / np.linalg.norm(d, axis=0, keepdims=True)).reshape(3, -1)               # camera.py:98-105

    def border_dirs64(self) -> np.ndarray:
        """Unit rays through the four image corners (camera.py:79-96,107-114): [3,4]."""
        t = np.array([[-1, 1, -1, 1], [-1, -1, 1, 1]], np.float64)
        d = np.stack([t[0] * self.width / 2.0 / self.focal, t[1] * self.height / 2.0 / self.focal, np.ones(4)])
        return d / np.linalg.norm(d, axis=0, keepdims=True)

    def cam_dirs(self, device) -> torch.Tensor:
        key = str(device)
        if key not in self._rays:
            self._rays[key] = torch.from_numpy(self._cam_dirs64()).float().to(device)      # camera.py:116-130
        return self._rays[key]

    def generate_rays(self, c2w: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """c2w [V,4,4] fp32 -> ray_dir [V,3,H,W], eye [V,3], z_dir [V,3] (camera.py:182-211, batched)."""
        rot = c2w[:, :3, :3]
        rays = torch.matmul(rot, self.cam_dirs(c2w.device)).reshape(-1, 3, self.height, self.width)
        return rays.contiguous(), c2w[:, :3, 3].contiguous(), rot[:, :, 2].contiguous()


class Camera:
    """The reference's general-intrinsics camera, same constructor / properties / `generate_rays` contract
    (gmpi/core/camera.py:13-211): K is any 3x3 upper-triangular intrinsic matrix (focal lengths, skew, principal point),
    `generate_rays(tf_c2w [4,4] numpy or torch, border_only)` -> (ray_dir [3,H,W] (or [3,2,2] for the image corners), eye [3],
    z_dir [3]), numpy in -> fp64 numpy out, torch in -> fp32 torch out.  K^-1 [u v 1] is evaluated in closed form (back
    substitution) instead of `np.linalg.inv` + matmul; the render path itself uses the batched `PinholeCamera`."""

    def __init__(self, height: int = 480, width: int = 640, intrinsics: np.ndarray = None, ray_from_pix_center: bool = False):
        assert intrinsics is not None and intrinsics.ndim == 2 and intrinsics.shape[0] == 3 and intrinsics.shape[1] == 3, (
            "[Camera] Expecting a 3x3 intrinsics matrix, but instead got {}".format(None if intrinsics is None else intrinsics.shape))
        self._h, self._w, self._K = height, width, intrinsics
        self._ray_from_pix_center = ray_from_pix_center
        self._cache = {}

    intrinsic_matrix = property(lambda self: self._K)
    height = property(lambda self: self._h)
    width = property(lambda self: self._w)

    def __repr__(self):
        return f"Camera: height={self.height}, width={self.width}, intrinsics=\n{self.intrinsic_matrix}"

    def _unproject(self, u: np.ndarray, v: np.ndarray) -> np.ndarray:
        """K^-1 [u v 1]^T by back substitution (K upper triangular): [3, ...] fp64."""
        K = np.asarray(self._K, np.float64)
        assert K[1, 0] == 0 and K[2, 0] == 0 and K[2, 1] == 0 and K[2, 2] != 0, "intrinsics must be upper triangular"
        z = 1.0 / K[2, 2]
        y = (v - K[1, 2] * z) / K[1, 1]
        x = (u - K[0, 1] * y - K[0, 2] * z) / K[0, 0]
        return np.stack(np.broadcast_arrays(x, y, np.full((1, 1), z)))

    @property
    def homogeneous_coordinates(self) -> np.ndarray:                    # [3,H,W], camera.py:53-76
        if "hom" not in self._cache:
            off = 0.5 if self._ray_from_pix_center else 0.0
            self._cache["hom"] = self._unproject(np.arange(int(self.width), dtype=np.float64)[None, :] + off,
                                                 np.arange(int(self.height), dtype=np.float64)[:, None] + off)
        return self._cache["hom"]

    @property
    def homogeneous_coordinates_border(self) -> np.ndarray:             # [3,2,2]: the image corners, camera.py:78-96
        if "homb" not in self._cache:
            self._cache["homb"] = self._unproject(np.array([[0.0, self.width]]), np.array([[0.0], [self.height]]))
        return self._cache["homb"]

    @staticmethod
    def _unit(d):
        return (d / np.linalg.norm(d, axis=0)).reshape(3, -1)

    ray_dir_np = property(lambda self: self._unit(self.homogeneous_coordinates))                   # [3,H*W] fp64, camera.py:98-105
    ray_dir_border_np = property(lambda self: self._unit(self.homogeneous_coordinates_border))     # [3,4]

    def _dirs_torch(self, device, border_only):
        key = (str(device), bool(border_only))
        if key not in self._cache:
            d = self.ray_dir_border_np if border_only else self.ray_dir_np
            self._cache[key] = torch.from_numpy(d).float().to(device)                              # camera.py:116-130
        return self._cache[key]

    ray_dir_torch = property(lambda self: self._dirs_torch("cpu", False))
    ray_dir_border_torch = property(lambda self: self._dirs_torch("cpu", True))

    def ray_dir_torch_cuda(self, device, border_only=False) -> torch.Tensor:
        return self._dirs_torch(device, border_only)

    def generate_rays(self, tf_c2w, border_only: bool = False):
        shape = (3, 2, 2) if border_only else (3, self.height, self.width)
        if isinstance(tf_c2w, np.ndarray):                                                         # camera.py:154-180
            rot = tf_c2w[:3, :3]
            return (rot @ (self.ray_dir_border_np if border_only else self.ray_dir_np)).reshape(shape), tf_c2w[:3, 3], rot[:, 2]
        if isinstance(tf_c2w, torch.Tensor):                                                       # camera.py:182-211
            rot = tf_c2w[:3, :3]
            return torch.matmul(rot, self._dirs_torch(tf_c2w.device, border_only)).reshape(shape), tf_c2w[:3, 3], rot[:, 2]
        raise ValueError


def gen_cam(*, h, w, f, ray_from_pix_center):
    """cam_utils.py:16-22: pinhole with the principal point at (w/2, h/2)."""
    return Camera(height=h, width=w, intrinsics=np.array([[f, 0.0, w / 2], [0.0, f, h / 2], [0.0, 0.0, 1.0]]),
                  ray_from_pix_center=ray_from_pix_center)


def cam_params(c2w: torch.Tensor, focal: float, height: int, width: int, ray_from_pix_center: bool = True) -> torch.Tensor:
    """[V,16] fp32 = {f0, f1, f2, pixel-centre offset, R row-major (9), eye (3)} per view: the `cam` input of the kernels' fast
    mode (rays generated in the kernel with PinholeCamera's arithmetic instead of uploading ray_dir [V,3,H,W]).  The focal
    length is an fp64 number (focal_from_fov); f0 + f1 + f2 is its exact three-piece fp32 expansion, so the kernel's fp64 camera
    ray is bit-identical to `_cam_dirs64`.  The principal point is (width/2, height/2), which the kernel derives itself."""
    V = c2w.shape[0]
    f = np.float64(focal)
    f0 = np.float32(f)
    f1 = np.float32(f - np.float64(f0))
    f2 = np.float32(f - np.float64(f0) - np.float64(f1))
    assert np.float64(f0) + np.float64(f1) + np.float64(f2) == f
    head = torch.tensor([float(f0), float(f1), float(f2), 0.5 if ray_from_pix_center else 0.0], dtype=torch.float32,
                        device=c2w.device).expand(V, 4)
    return torch.cat([head, c2w[:, :3, :3].reshape(V, 9).float(), c2w[:, :3, 3].float()], dim=1).contiguous()


def truncated_normal(n: int, mean: float, std: float, n_std: float, generator: Optional[torch.Generator] = None):
    """Draw 4 normals per sample and keep the first inside mean +- n_std*std (gmpi/utils/torch_utils.py:51-76)."""
    tmp = torch.randn((n, 1, 4), generator=generator) * std + mean
    lo, hi = mean - n_std * std, mean + n_std * std
    ok = (tmp < hi) & (tmp > lo)
    first = ok.float().argmax(-1, keepdim=True)
    return tmp.gather(-1, first).squeeze(-1).clamp(lo, hi)


def sphere_poses(yaws: torch.Tensor, pitches: torch.Tensor, sphere_center, sphere_r: float = 1.0) -> torch.Tensor:
    """Camera-to-world matrices [V,4,4] (fp32 values) for cameras on the sphere looking at its centre.

    Sphere frame (+X back, +Y right, +Z up): p = r(|cos pitch| cos yaw, |cos pitch| sin yaw, sin pitch)
    (cam_utils.py:561-564); forward = -p/|p|; right = down0 x forward with down0 = (0,0,-1); down = forward x
    right (cam_utils.py:571-622).  Sphere -> world maps (x,y,z) to (y,-z,-x) + centre, i.e. Rx(90deg) Rz(-90deg)
    then the translation (cam_utils.py:687-731)."""
    yaws = yaws.reshape(-1, 1).float()
    pitches = pitches.reshape(-1, 1).float()
    rc = sphere_r * torch.abs(torch.cos(pitches))
    pos = torch.cat([rc * torch.cos(yaws), rc * torch.sin(yaws), sphere_r * torch.sin(pitches)], 1)    # fp32, in the reference's order
    unit = lambda v: v / torch.norm(v, dim=-1, keepdim=True)
    fwd = unit(unit(-pos))                                            # normalised twice, as the reference does (cam_utils.py:786, :599)
    down0 = torch.tensor([0.0, 0.0, -1.0]).expand_as(fwd)
    right = unit(torch.cross(down0, fwd, dim=-1))
    down = unit(torch.cross(fwd, right, dim=-1))
    c2s = torch.eye(4).repeat(pos.shape[0], 1, 1)
    c2s[:, :3, :3] = torch.stack((right, down, fwd), dim=-1)
    c2s[:, :3, 3] = pos
    s2w = np.array([[0, 1, 0, 0], [0, 0, -1, 0], [-1, 0, 0, 0], [0, 0, 0, 1]], np.float64)
    s2w[:3, 3] = np.asarray(sphere_center, np.float64).reshape(-1)
    return torch.from_numpy(np.matmul(s2w, c2s.numpy().astype(np.float64))).float()                    # cam_utils.py:798, :364


def sample_yaw_pitch(n, h_mean, h_std, v_mean, v_std, n_std=2, method="truncated_gaussian", random_pose=True,
                     horizontal_sweep=True, generator=None):
    """Pose angles as sample_camera_positions_sphere draws them (cam_utils.py:510-555)."""
    if random_pose:
        if method == "uniform":
            y = (torch.rand((n, 1), generator=generator) - 0.5) * 2 * n_std * h_std + h_mean
            p = (torch.rand((n, 1), generator=generator) - 0.5) * 2 * n_std * v_std + v_mean
        elif method in ("normal", "gaussian"):
            y = torch.randn((n, 1), generator=generator) * h_std + h_mean
            p = torch.randn((n, 1), generator=generator) * v_std + v_mean
        elif method == "truncated_gaussian":
            y = truncated_normal(n, h_mean, h_std, n_std, generator)
            p = truncated_normal(n, v_mean, v_std, n_std, generator)
        else:
            raise ValueError(method)
    elif horizontal_sweep:
        y = torch.linspace(-n_std, n_std, n).reshape(n, 1) * h_std + h_mean
        p = torch.ones((n, 1)) * v_mean
    else:
        y = torch.ones((n, 1)) * h_mean
        p = torch.linspace(-n_std, n_std, n).reshape(n, 1) * v_std + v_mean
    return y, p
