"""8-bit plane-image fixture (tests/test_unorm8.py, tests/test_gpu_unorm8.py): an MPI built by the UNMODIFIED reference's
mpi_from_plane_imgs (gmpi/utils/mpi_utils.py:302-357) from seeded RGBA8 plane images, and the reference MPI.forward's render of it,
produced on CPU:

    python oracle/make_golden_u8.py      # needs /root/reference; writes tests/golden/u8_planes.npz

mpi_from_plane_imgs converts each uint8 plane with astype(np.float32) / 255.0 and stacks the planes front to back as [N,4,h,w].  The
fixture keeps the same planes as the planar uint8 tensor [1,N,4,h,w] (rgba_u8, front to back), the reference's fp32 MPI (rgba),
its plane table (dhw) and the reference render from three FFHQ poses (color, depth).  The planes have transparent regions (alpha 0)
and a wide range of alpha codes.

Layout: rgba_u8 [1,N,4,h,w] uint8, rgba [1,N,4,h,w] float32, dhw [1,N,3], view2mpi [V], ray_dir [V,3,H,W], eye [V,3], z_dir [V,3],
align_corners (bool), color [V,3,H,W], depth [V,1,H,W].

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
from make_golden import cams, make_renderer, pack_views, save  # noqa: E402

N, TEX_H, TEX_W, IMG = 8, 64, 80, 64


def plane_images(seed):
    """N RGBA8 plane images [h, w, 4], back to front (mpi_from_plane_imgs' order): random colour, alpha random inside a disc per plane
    (0 outside it), the furthest plane opaque."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:TEX_H, 0:TEX_W]
    out = []
    for k in range(N):
        img = rng.integers(0, 256, (TEX_H, TEX_W, 4), dtype=np.uint8)
        cy, cx, r = rng.uniform(0.3, 0.7) * TEX_H, rng.uniform(0.3, 0.7) * TEX_W, rng.uniform(0.2, 0.45) * TEX_H
        img[..., 3][(yy - cy) ** 2 + (xx - cx) ** 2 > r * r] = 0
        if k == 0:
            img[..., 3] = 255
        out.append(img)
    return out


def main():
    torch.set_num_threads(8)
    ref_mpi, ref_r = ref_shim.import_reference()
    import gmpi.utils.mpi_utils as ref_mpi_utils       # noqa: E402  (importable once the shims are installed)
    imgs = plane_images(5)
    with contextlib.redirect_stdout(io.StringIO()):
        planes, dhws, _ = ref_mpi_utils.mpi_from_plane_imgs(dmin=0.9, dmax=1.1, plane_rgbas=[im.copy() for im in imgs])
    # the same planes as one planar uint8 tensor, front to back (the function reverses its list in place)
    rgba_u8 = np.stack([im.transpose(2, 0, 1) for im in imgs[::-1]])[None]
    rgba = planes.numpy()[None].astype(np.float32)
    dhw = dhws.numpy().astype(np.float32)[None]
    r = make_renderer(ref_r, N)
    c = cams(r, IMG, [-0.25, 0.0, 0.3], [0.1, -0.05, 0.0])
    groups = tuple([torch.cat(list(c[k]))] for k in ("batch_ray_dir", "batch_eye_pos", "batch_z_dir"))   # one MPI, three views
    mod = ref_mpi.MPI(align_corners=True)
    with torch.no_grad(), contextlib.redirect_stdout(io.StringIO()):
        color, depth = mod(batch_rgba=torch.from_numpy(rgba), batch_dhw=torch.from_numpy(dhw), batch_ray_dir=groups[0],
                           batch_eye_pos=groups[1], batch_z_dir=groups[2], separate_background=None, assert_not_out_of_last_plane=False)
    save("u8_planes", rgba_u8=rgba_u8, rgba=rgba, dhw=dhw, align_corners=np.bool_(True), color=color.numpy(), depth=depth.numpy(),
         **pack_views(*groups))


if __name__ == "__main__":
    main()
