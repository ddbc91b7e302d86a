"""Synthetic MPI workloads with the reference's FFHQ geometry (SURVEY.md section 8d), or another dataset's (geometry.AFHQCAT,
geometry.METFACES): random RGBA stacks, in-envelope poses, rays from the pinhole camera.  Used by bench.py, smoke() and the
full-size GPU tests; needs neither the reference nor the oracle."""
from dataclasses import dataclass

import numpy as np
import torch

from .camera import PinholeCamera, sphere_poses
from .geometry import FFHQ, plane_dhw_table

_DHW_CACHE = {}


def plane_table(n_planes: int, geometry=FFHQ) -> torch.Tensor:
    """The [n_planes, 3] plane table of a geometry (geometry.FFHQ, AFHQCAT, METFACES), built once per geometry and plane count."""
    key = (n_planes,) + tuple(sorted(geometry.items()))
    if key not in _DHW_CACHE:
        _DHW_CACHE[key] = torch.from_numpy(plane_dhw_table(n_planes=n_planes, **geometry))
    return _DHW_CACHE[key]


def ffhq_dhw(n_planes: int) -> torch.Tensor:
    return plane_table(n_planes, FFHQ)


@dataclass
class Case:
    rgba: torch.Tensor       # [M,N,4,T,T]
    dhw: torch.Tensor        # [M,N,3]
    view2mpi: torch.Tensor   # [V] int32
    ray_dir: torch.Tensor    # [V,3,H,W]
    eye: torch.Tensor        # [V,3]
    z_dir: torch.Tensor      # [V,3]
    c2w: torch.Tensor        # [V,4,4]
    yaws: torch.Tensor
    pitches: torch.Tensor

    def to(self, device, pin=False):
        f = (lambda t: t.pin_memory()) if pin else (lambda t: t.to(device))
        return Case(*[f(getattr(self, k)) for k in self.__dataclass_fields__])


def make_poses(n_views, img, seed=1234, yaws=None, pitches=None, device="cpu", geometry=FFHQ):
    """Rays of n_views poses on the geometry's camera sphere, with its fov.  Without yaws / pitches: U(-0.5,0.5) x U(-0.2,0.2),
    inside FFHQ's 2-sigma envelope (BASELINE.md section 4), whatever the geometry."""
    if yaws is None:
        rng = np.random.default_rng(seed)
        yaws = rng.uniform(-0.5, 0.5, n_views).astype(np.float32)
        pitches = rng.uniform(-0.2, 0.2, n_views).astype(np.float32)
    yaws, pitches = torch.as_tensor(yaws, dtype=torch.float32), torch.as_tensor(pitches, dtype=torch.float32)
    c2w = sphere_poses(yaws, pitches, geometry["sphere_center"], geometry["sphere_r"]).to(device)
    cam = PinholeCamera.from_fov(geometry["fov_deg"], img, img)
    ray_dir, eye, z_dir = cam.generate_rays(c2w)
    return ray_dir, eye, z_dir, c2w, yaws, pitches


def envelope_poses(geometry=FFHQ, scale=1.0):
    """(yaws, pitches) fp32 [9] at the edge of the geometry's truncated-Gaussian pose envelope, mean +- n_truncated_stds x std
    (what the plane table is sized for, geometry.plane_dhw_table), times `scale`: the four corners (-,-), (+,-), (-,+), (+,+), then
    the four edge midpoints (-,0), (+,0), (0,-), (0,+), then the centre."""
    k = geometry["n_truncated_stds"] * scale
    hy, hp = k * geometry["h_std"], k * geometry["v_std"]
    sy = [-1, 1, -1, 1, -1, 1, 0, 0, 0]
    sp = [-1, -1, 1, 1, 0, 0, -1, 1, 0]
    yaws = np.array([geometry["h_mean"] + s * hy for s in sy], np.float32)
    pitches = np.array([geometry["v_mean"] + s * hp for s in sp], np.float32)
    return yaws, pitches


def make_case(*, n_planes, tex, img, n_mpi, views_per_mpi=1, seed=1234, device="cpu", last_alpha_one=False,
              yaws=None, pitches=None, rgba=True, alpha="uniform", geometry=FFHQ) -> Case:
    """alpha: "uniform" (U(0, 1) on every plane) or "equal_weight" (equal_weight_alpha, whose last plane is opaque).
    geometry: the plane table, camera sphere and fov (geometry.FFHQ, AFHQCAT, METFACES)."""
    assert alpha in ("uniform", "equal_weight"), alpha
    V = n_mpi * views_per_mpi
    ray_dir, eye, z_dir, c2w, yaws, pitches = make_poses(V, img, seed, yaws, pitches, device, geometry)
    gen = torch.Generator(device=device).manual_seed(seed)
    t = None
    if rgba:
        t = torch.rand((n_mpi, n_planes, 4, tex, tex), generator=gen, device=device, dtype=torch.float32)
        if alpha == "equal_weight":
            t[:, :, 3] = equal_weight_alpha((n_mpi, n_planes, tex, tex), gen, device)
        if last_alpha_one:
            t[:, -1, 3] = 1.0      # production MPIs: networks_cond_on_pos_enc.py:1307-1310
    dhw = plane_table(n_planes, geometry).to(device).unsqueeze(0).expand(n_mpi, -1, -1).contiguous()
    v2m = torch.arange(n_mpi, dtype=torch.int32, device=device).repeat_interleave(views_per_mpi)
    return Case(t, dhw, v2m, ray_dir, eye, z_dir, c2w, yaws, pitches)


def equal_weight_alpha(shape, generator, device="cpu") -> torch.Tensor:
    """[..., N, Ht, Wt] alpha under which every plane carries weight: U(0, 1) alpha hides the planes past ~25 (transmittance
    falls as e^-i), so a render or gradient check at 96 planes could not see a kernel error on them.  Plane i gets
    min(1, u * 2 / (N - i)), u ~ U(0, 1) per texel (E[alpha_i] = 1 / (N - i), hence an expected compositing weight of 1 / N for
    every plane), and the last plane is opaque, as in a GMPI MPI."""
    n = shape[-3]
    u = torch.rand(shape, generator=generator, device=device, dtype=torch.float32)
    scale = 2.0 / torch.arange(n, 0, -1, device=device, dtype=torch.float32)
    alpha = torch.clamp(u * scale[:, None, None], max=1.0)
    alpha[..., -1, :, :] = 1.0
    return alpha


def head_alpha(n_planes: int, tex: int, device="cpu") -> torch.Tensor:
    """[N,T,T] alpha of a structured synthetic MPI: a transparent volume with an opaque ellipsoidal "head" (semi-axes 0.8 x 0.95
    of the texture, about 60 % of the frame) whose front surface crosses K = max(2, N // 16) planes around the middle, plus the
    alpha == 1 last plane of a GMPI MPI (networks_cond_on_pos_enc.py:1307-1310).  Plane c0 + k is opaque where the surface lies in
    front of or on it (a disc that widens with depth), so pixels stop at different planes and the rim (partial bilinear alpha)
    stays transparent until the last plane.  A trained MPI has not been measured against it."""
    K = max(2, n_planes // 16)
    c0 = max(0, n_planes // 2 - K // 2)
    ax = torch.linspace(-1.0, 1.0, tex, device=device)
    y, x = torch.meshgrid(ax, ax, indexing="ij")
    r2 = (x / 0.8) ** 2 + (y / 0.95) ** 2
    depth = (1.0 - torch.sqrt(torch.clamp(1.0 - r2, min=0.0))) * K      # front surface, in planes behind c0
    alpha = torch.zeros((n_planes, tex, tex), device=device)
    for k in range(K):
        if c0 + k < n_planes:
            alpha[c0 + k] = ((r2 < 1.0) & (depth < k + 1)).float()
    alpha[-1] = 1.0
    return alpha


def make_head_case(*, n_planes, tex, img, n_mpi, views_per_mpi=1, seed=1234, device="cpu", yaws=None, pitches=None,
                   geometry=FFHQ) -> Case:
    """make_case with random colours and head_alpha's alpha (tools/early_stop_bench.py and the early-stop tests)."""
    case = make_case(n_planes=n_planes, tex=tex, img=img, n_mpi=n_mpi, views_per_mpi=views_per_mpi, seed=seed, device=device,
                     yaws=yaws, pitches=pitches, rgba=False, geometry=geometry)
    gen = torch.Generator(device=device).manual_seed(seed)
    rgba = torch.rand((n_mpi, n_planes, 4, tex, tex), generator=gen, device=device, dtype=torch.float32)
    rgba[:, :, 3] = head_alpha(n_planes, tex, device)
    case.rgba = rgba
    return case
