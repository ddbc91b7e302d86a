#!/usr/bin/env python
"""Does a memset of the gradient overlap a persistent kernel?  CUDA-event times on the headline train shape (4 MPIs x 1 view,
96 planes, 1024^2): the training-mode forward alone, a memset of the gradient alone, and both at once on two streams.
python tools/zero_overlap_probe.py"""
import sys

import torch

sys.path.insert(0, ".")
import ml_gmpi_b200 as g                     # noqa: E402
from ml_gmpi_b200 import _lib, synth         # noqa: E402

dev = torch.device("cuda:0")
case = synth.make_case(device=dev, n_mpi=4, views_per_mpi=1, n_planes=96, tex=1024, img=1024, seed=0)
rg = case.rgba.requires_grad_(True)
lib = _lib.load()
side = torch.cuda.Stream(device=dev)
main = torch.cuda.current_stream(dev)
buf = torch.empty_like(case.rgba)


def timed(fn, n=6, warm=2):
    ts = []
    for i in range(warm + n):
        torch.cuda.synchronize(dev)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        side.wait_stream(main)
        a.record(main)
        fn()
        main.wait_stream(side)
        b.record(main)
        torch.cuda.synchronize(dev)
        if i >= warm:
            ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


def fwd():
    return g.render_views(rg, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, color_minus1_1=True)[0]


def zero_side():
    _lib.check(lib.gmpi_mpi_zero_async(buf.data_ptr(), buf.numel() * 4, side.cuda_stream))


def both():
    zero_side()
    fwd()


t_fwd, t_zero, t_both = timed(fwd), timed(zero_side), timed(both)
print(f"forward(train) alone {t_fwd:.3f} ms; memset alone {t_zero:.3f} ms; both on two streams {t_both:.3f} ms (sum {t_fwd + t_zero:.3f})")
