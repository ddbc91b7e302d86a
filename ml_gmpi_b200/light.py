"""Mirror of `gmpi.core.light_renderer.LightRenderer` (gmpi/core/light_renderer.py:11-199), the lighting augmentation the
training loop applies to the MPI right before `MPIRenderer.render` (train.py:534-541,702-709) -- SURVEY.md 8(f) row N3.

Same constructor keywords, same methods (`get_normal`, `compute_depth`, `compute_pcl`, `render`), same step-dependent
ka/kd growth.  What moves to CUDA (csrc/mpi_light.cuh, through the C ABI):
  * `compute_depth` (:82-100): the renderer's over-composite on the un-warped alpha.  The reference builds
    [B,N+1,1,H,W] (cat), its cumprod, the weights and weights*plane_ds -- five full-size tensors; here one streaming
    kernel (4 B per texel-plane) with its own backward (autograd.Function, first order);
  * the last step of `render` (:190-199): `clip(rgb*shading, 0, 1)` + `cat` -> one fused pass producing the new MPI.
The Gaussian blur, the point cloud, the normals and the Lambertian term act on [B,H,W] images (1/N of the MPI) and stay
torch ops -- plumbing on small tensors.  With the generator's FACTORED output the shading step is a [B,3,H,W] product:
`shade_factored` returns the shaded colour image and the renderer consumes (rgb, alpha) directly (render_views_factored).
Both kernels stream four texels per thread; a texture whose Ht*Wt is not a multiple of 4 takes the reference's fp32 torch
expressions instead (the C ABI refuses such sizes).

No CPU path: tensors must live on a CUDA device.
"""
from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F

from . import _lib
from .camera import sample_yaw_pitch, sphere_poses
from .mpi import _require_cuda, _stream_ptr

EPS = 1e-8          # light_renderer.py:8


def _streamable(t: torch.Tensor) -> torch.Tensor:
    """t as a contiguous fp32 tensor whose base is 16-byte aligned, as the float4 kernels read it: t itself when it already is,
    else a copy (a contiguous view that starts mid-allocation, e.g. one float in, is copied too)."""
    t = t.float().contiguous()
    return t if t.data_ptr() % 16 == 0 else t.clone()


def _alpha_view(mpi_alpha: torch.Tensor):
    """(tensor to keep alive, base pointer, mpi_stride, plane_stride) of an alpha stack [B,N,1,H,W]: a contiguous tensor, or the
    channel-3 view of a contiguous [B,N,4,H,W] stack (no copy)."""
    B, N, _, H, W = mpi_alpha.shape
    st = mpi_alpha.stride()
    if mpi_alpha.dtype == torch.float32 and st[-1] == 1 and st[-2] == W and st[1] % 4 == 0 and st[0] % 4 == 0 and \
            mpi_alpha.data_ptr() % 16 == 0 and (H * W) % 4 == 0:
        return mpi_alpha, mpi_alpha.data_ptr(), st[0], st[1]
    c = _streamable(mpi_alpha)
    return c, c.data_ptr(), N * H * W, H * W


class _AlphaDepthFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mpi_alpha, plane_ds, save_t):
        lib = _lib.load()
        B, N, _, H, W = mpi_alpha.shape
        keep, ptr, ms, ps = _alpha_view(mpi_alpha)
        depth = torch.empty((B, 1, H, W), device=mpi_alpha.device, dtype=torch.float32)
        trans = torch.empty((B, N, H, W), device=mpi_alpha.device, dtype=torch.float32) if save_t else None
        with torch.cuda.device(mpi_alpha.device):
            _lib.check(lib.gmpi_mpi_alpha_depth_fwd(ptr, ms, ps, plane_ds.data_ptr(), depth.data_ptr(),
                                                    None if trans is None else trans.data_ptr(), B, N, H, W,
                                                    _stream_ptr(mpi_alpha.device)))
        ctx.save_for_backward(keep, plane_ds, trans)
        ctx.view = (ms, ps)
        return depth

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_depth):
        keep, plane_ds, trans = ctx.saved_tensors
        if trans is None:
            return None, None, None
        lib = _lib.load()
        B, N, H, W = trans.shape
        ms, ps = ctx.view
        g_alpha = torch.empty((B, N, 1, H, W), device=trans.device, dtype=torch.float32)
        g = g_depth.float().contiguous()
        with torch.cuda.device(trans.device):
            _lib.check(lib.gmpi_mpi_alpha_depth_bwd(keep.data_ptr() if keep.is_contiguous() else keep.data_ptr(), ms, ps,
                                                    plane_ds.data_ptr(), trans.data_ptr(), g.data_ptr(), g_alpha.data_ptr(),
                                                    N * H * W, H * W, B, N, H, W, _stream_ptr(trans.device)))
        return g_alpha, None, None


class _ApplyShadingFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, rgba, shade):
        lib = _lib.load()
        B, N, _, H, W = rgba.shape
        out = torch.empty_like(rgba)
        with torch.cuda.device(rgba.device):
            _lib.check(lib.gmpi_mpi_apply_shading_fwd(rgba.data_ptr(), shade.data_ptr(), out.data_ptr(), B, N, H, W, _stream_ptr(rgba.device)))
        ctx.save_for_backward(rgba, shade)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    def backward(ctx, g_out):
        rgba, shade = ctx.saved_tensors
        lib = _lib.load()
        B, N, _, H, W = rgba.shape
        g_rgba, g_shade = torch.empty_like(rgba), torch.empty_like(shade)
        g = g_out.float().contiguous()
        with torch.cuda.device(rgba.device):
            _lib.check(lib.gmpi_mpi_apply_shading_bwd(rgba.data_ptr(), shade.data_ptr(), g.data_ptr(), g_rgba.data_ptr(),
                                                      g_shade.data_ptr(), B, N, H, W, _stream_ptr(rgba.device)))
        return g_rgba, g_shade


def alpha_depth(mpi_alpha: torch.Tensor, plane_ds: torch.Tensor) -> torch.Tensor:
    """LightRenderer.compute_depth (light_renderer.py:82-100): [B,N,1,H,W] alpha, [N] plane distances -> [B,1,H,W]."""
    _require_cuda(mpi_alpha, "ml_gmpi_b200 runs")
    pd = plane_ds.reshape(-1).to(device=mpi_alpha.device, dtype=torch.float32).contiguous()
    B, N, _, H, W = mpi_alpha.shape
    assert pd.numel() == N, f"{mpi_alpha.shape}, {plane_ds.shape}"
    if (H * W) % 4:
        # the kernel streams four texels per thread; other texel counts take the reference's fp32 expression and its autograd
        a = mpi_alpha.float()[:, :, 0]
        s = (1.0 - a) + 1e-10
        trans = torch.cumprod(torch.cat((torch.ones_like(s[:, :1]), s[:, :-1]), dim=1), dim=1)
        return (a * trans * pd.view(1, N, 1, 1)).sum(1, keepdim=True)
    # T (4 B per texel-plane) is only needed by a backward, and grad mode is always off inside Function.forward: decide here
    return _AlphaDepthFn.apply(mpi_alpha, pd, torch.is_grad_enabled() and mpi_alpha.requires_grad)


def apply_shading(batch_mpi: torch.Tensor, shading: torch.Tensor) -> torch.Tensor:
    """clip(rgb * shading, 0, 1) on the colour channels, alpha unchanged (light_renderer.py:190-199): [B,N,4,H,W] x [B,1,H,W]."""
    _require_cuda(batch_mpi, "ml_gmpi_b200 runs")
    B, N, C, H, W = batch_mpi.shape
    assert C == 4, f"{batch_mpi.shape}"
    if (H * W) % 4:
        # as in alpha_depth: texel counts the float4 kernel cannot stream take the reference's fp32 expression.  split (not two
        # slices) so that d rgb is g * shade as the kernel writes it: slices would add a zero-filled alpha gradient, turning -0 into +0
        rgb, alpha = batch_mpi.float().split((3, 1), dim=2)
        return torch.cat((torch.clip(rgb * shading.reshape(B, 1, 1, H, W).float(), min=0.0, max=1.0), alpha), dim=2)
    return _ApplyShadingFn.apply(_streamable(batch_mpi), _streamable(shading.reshape(B, 1, H, W)))


def gaussian_blur(img: torch.Tensor, ksize: int, sigma: float) -> torch.Tensor:
    """torchvision.transforms.GaussianBlur(kernel_size, sigma) on [B,1,H,W] (light_renderer.py:50-53): separable kernel
    exp(-x^2 / (2 sigma^2)) over linspace(-(k-1)/2, (k-1)/2, k), normalised, reflect padding, one 2-D convolution."""
    half = (ksize - 1) * 0.5
    x = torch.linspace(-half, half, steps=ksize, device=img.device, dtype=img.dtype)
    pdf = torch.exp(-0.5 * (x / sigma).pow(2))
    k1 = pdf / pdf.sum()
    k2 = torch.mm(k1[:, None], k1[None, :])
    pad = ksize // 2
    x = F.pad(img, [pad, pad, pad, pad], mode="reflect")
    return F.conv2d(x, k2[None, None].expand(img.shape[1], 1, ksize, ksize), groups=img.shape[1])


class LightRenderer:
    def __init__(self, *, sphere_center_z, sphere_r, ka_max=1.0, kd_max=0.0, n_grow_iters=1000, l_h_mean=0.0, l_h_std=0.2,
                 l_v_mean=0.2, l_v_std=0.05, blur_ksize=9):
        self.ka_max, self.kd_max, self.n_grow_iters = ka_max, kd_max, n_grow_iters
        self.cur_ka, self.cur_kd = 0.0, 0.0
        self.l_h_mean, self.l_h_std, self.l_v_mean, self.l_v_std = l_h_mean, l_h_std, l_v_mean, l_v_std
        self.sphere_center = torch.FloatTensor(np.array([0, 0, sphere_center_z]))
        self.sphere_r = sphere_r
        self.blur_ksize = blur_ksize
        self.blur_sigma = 0.3 * ((self.blur_ksize - 1) * 0.5 - 1) + 0.8          # light_renderer.py:49
        self.step = -1

    # light_renderer.py:57-80
    def get_normal(self, grid_3d, normalize=True):
        center = grid_3d[:, 1:-1, 1:-1]
        up, down, left, right = grid_3d[:, :-2, 1:-1], grid_3d[:, 2:, 1:-1], grid_3d[:, 1:-1, :-2], grid_3d[:, 1:-1, 2:]
        normal = (torch.cross(up - center, left - center, dim=3) + torch.cross(left - center, down - center, dim=3)
                  + torch.cross(down - center, right - center, dim=3) + torch.cross(right - center, up - center, dim=3))
        normal = F.pad(normal.permute(0, 3, 1, 2), (1, 1, 1, 1), mode="replicate").permute(0, 2, 3, 1)
        if normalize:
            normal = normal / (((normal ** 2).sum(3, keepdim=True)) ** 0.5 + EPS)
        return normal

    # light_renderer.py:82-100
    def compute_depth(self, mpi_alpha, plane_ds):
        return alpha_depth(mpi_alpha, plane_ds)

    # light_renderer.py:102-120
    def compute_pcl(self, mpi_alpha, mpi_plane_dhws, mpi_tex_pix_xyz):
        plane_ds = mpi_plane_dhws[:, :1].to(mpi_alpha.device)
        mpi_depth = self.compute_depth(mpi_alpha, plane_ds)
        mpi_depth = self._blur(mpi_depth)[:, 0, ...]
        mpi_xyz_last_plane = mpi_tex_pix_xyz[-1:, :, :, :3]
        scale = mpi_depth.unsqueeze(-1) / (mpi_xyz_last_plane[..., 2:] + EPS)
        return mpi_xyz_last_plane * scale

    def _blur(self, img):
        """The reference blurs with torchvision.transforms.GaussianBlur(sigma=(s, s)) (light_renderer.py:50-53,112), whose forward
        draws its sigma with torch.empty(1).uniform_(s, s) -- ONE value of torch's global CPU generator per call, BEFORE the light is
        sampled.  The draw is repeated here (its value is s whatever the generator returns) so that a seeded run sees the same
        random stream -- the same lights, and the same poses and latents afterwards -- as with the reference."""
        torch.empty(1).uniform_(self.blur_sigma, self.blur_sigma)
        return gaussian_blur(img, self.blur_ksize, self.blur_sigma)

    def sample_light_directions(self, bs, device, given_yaws=None, given_pitches=None):
        """Light position on the camera sphere, direction towards its centre (light_renderer.py:136-165)."""
        if given_yaws is None:
            given_yaws, given_pitches = sample_yaw_pitch(bs, self.l_h_mean, self.l_h_std, self.l_v_mean, self.l_v_std, 2,
                                                         "truncated_gaussian", True)
        c2w = sphere_poses(given_yaws.cpu(), given_pitches.cpu(), self.sphere_center.numpy(), self.sphere_r)
        light_pos = c2w[:, :3, 3].to(device)
        d = self.sphere_center.reshape((1, 3)).to(device) - light_pos
        return d / torch.norm(d, dim=-1, keepdim=True)                         # normalize_vecs, torch_utils.py

    def shading(self, mpi_alpha, mpi_plane_dhws, mpi_tex_pix_xyz, given_yaws=None, given_pitches=None):
        """[B,1,1,H,W] Lambertian shading of this step (light_renderer.py:133-188); advances `step`."""
        self.step += 1
        bs = mpi_alpha.shape[0]
        grid_3d = self.compute_pcl(mpi_alpha, mpi_plane_dhws, mpi_tex_pix_xyz)
        light_direction = self.sample_light_directions(bs, mpi_alpha.device, given_yaws, given_pitches)
        canon_normal = self.get_normal(grid_3d)
        diffuse = (-1 * (canon_normal * light_direction.view(-1, 1, 1, 3)).sum(3)).clamp(min=0)
        diffuse = diffuse.unsqueeze(1).unsqueeze(1)
        cur_ratio = min(1.0, self.step / self.n_grow_iters)
        self.cur_ka, self.cur_kd = cur_ratio * self.ka_max, cur_ratio * self.kd_max
        ka = torch.ones((bs,), device=mpi_alpha.device) * self.cur_ka
        kd = torch.ones((bs,), device=mpi_alpha.device) * self.cur_kd
        return ka.view((bs, 1, 1, 1, 1)) + diffuse * kd.view((bs, 1, 1, 1, 1))

    # light_renderer.py:122-199
    def render(self, batch_mpi, mpi_plane_dhws, mpi_tex_pix_xyz, given_yaws: Optional[torch.Tensor] = None,
               given_pitches: Optional[torch.Tensor] = None):
        """[B,N,4,H,W] -> the shaded MPI, same shape.  `given_yaws/pitches` ([B,1]) fix the light (the reference always samples)."""
        canon_shading = self.shading(batch_mpi[:, :, 3:, ...], mpi_plane_dhws, mpi_tex_pix_xyz, given_yaws, given_pitches)
        return apply_shading(batch_mpi, canon_shading[:, 0])

    def shade_factored(self, rgb, alpha, mpi_plane_dhws, mpi_tex_pix_xyz, given_yaws=None, given_pitches=None):
        """Factored MPI (rgb [B,3,H,W] shared by all planes, alpha [B,N,1,H,W]): the shaded colour image.  Equal to
        `render(expand(rgb, alpha))[:, i, :3]` for every plane i -- the shading does not depend on the plane."""
        canon_shading = self.shading(alpha, mpi_plane_dhws, mpi_tex_pix_xyz, given_yaws, given_pitches)
        return torch.clip(rgb * canon_shading[:, 0], min=0.0, max=1.0)
