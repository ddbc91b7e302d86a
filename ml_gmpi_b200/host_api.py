"""End-to-end entry point on HOST buffers (pinned memory recommended): wraps gmpi_mpi_render_fwd_host of the
C ABI, which streams the MPIs through a double-buffered device staging area (copy of MPI m+1 overlaps the render
of MPI m) and returns colour/depth in host memory."""
import numpy as np
import torch

from . import _lib
from .mpi import _options


def render_host(rgba: torch.Tensor, dhw: torch.Tensor, view2mpi: torch.Tensor, ray_dir: torch.Tensor, eye: torch.Tensor,
                z_dir: torch.Tensor, *, align_corners=True, check_last_plane=False, color_minus1_1=False, device=0,
                out_color: torch.Tensor = None, out_depth: torch.Tensor = None):
    """All inputs are CPU tensors (fp32 contiguous; int32 view2mpi sorted MPI-major).  Returns
    (color [V,3,H,W], depth [V,1,H,W], flags:int) as CPU tensors (pinned if the outputs are passed pinned)."""
    for t in (rgba, dhw, ray_dir, eye, z_dir):
        assert t.device.type == "cpu" and t.dtype == torch.float32 and t.is_contiguous()
    assert view2mpi.device.type == "cpu" and view2mpi.dtype == torch.int32
    lib = _lib.load()
    M, N, _, Ht, Wt = rgba.shape
    V, _, H, W = ray_dir.shape
    if out_color is None:
        out_color = torch.empty((V, 3, H, W), dtype=torch.float32).pin_memory()
    if out_depth is None:
        out_depth = torch.empty((V, 1, H, W), dtype=torch.float32).pin_memory()
    flags = np.zeros(1, np.uint32)
    options = _options(align_corners, check_last_plane, color_minus1_1)
    _lib.check(lib.gmpi_mpi_render_fwd_host(rgba.data_ptr(), view2mpi.data_ptr(), dhw.data_ptr(), ray_dir.data_ptr(),
                                            eye.data_ptr(), z_dir.data_ptr(), out_color.data_ptr(), out_depth.data_ptr(),
                                            flags.ctypes.data, M, V, N, Ht, Wt, H, W, options, int(device)))
    return out_color, out_depth, int(flags[0])
