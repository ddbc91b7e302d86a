#!/usr/bin/env python
"""Forward time with and without early ray termination (GMPI_EARLY_STOP) on a STRUCTURED synthetic MPI:
    python tools/early_stop_bench.py [--tau 5.96e-8] [--rounds 5] [--steps 20]
The workload is synth.make_head_case (a transparent volume, an opaque ellipsoidal head over ~60 % of the frame crossing a few
middle planes, alpha == 1 last plane) at two shapes: 4 MPIs x 1 view, 96 planes, 1024^2 (bench.py's headline shape) and the 512^2
video sweep (120 views of one 96-plane MPI, views grouped).  bench.py's random-alpha inputs make T < 2^-24 within ~17 planes, so
an early-stop number on them would say nothing about real MPIs; this synthetic MPI is not a trained one either.  Off and on
alternate within every round; prints one JSON line with the medians, the share of (tile, plane) stages whose loads were skipped
(gmpi_debug_fwd_early_stop_stats) and the largest colour change (bound: 2 tau in [-1,1]).  Writes nothing."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch
from ml_gmpi_b200 import _lib, synth


def measure(case, view_group, tau, rounds, steps):
    lib = _lib.load()
    V, _, H, W = case.ray_dir.shape
    M, N, _, Ht, Wt = case.rgba.shape
    dev = case.rgba.device
    color, depth = torch.empty((V, 3, H, W), device=dev), torch.empty((V, 1, H, W), device=dev)
    flags = torch.zeros(1, dtype=torch.int32, device=dev)
    st = torch.cuda.current_stream(dev).cuda_stream
    base = _lib.OPT_ALIGN_CORNERS | _lib.OPT_CHECK_LAST_PLANE | _lib.OPT_COLOR_MINUS1_1
    descs = {}
    for name, es in (("off", None), ("early_stop", tau)):
        descs[name] = _lib.make_desc(options=base | (_lib.OPT_EARLY_STOP if es is not None else 0), early_stop=es, M=M, V=V, N=N,
                                     Ht=Ht, Wt=Wt, H=H, W=W, view_group=view_group, rgba=case.rgba, view2mpi=case.view2mpi,
                                     dhw=case.dhw, ray_dir=case.ray_dir, eye=case.eye, z_dir=case.z_dir, color=color, depth=depth,
                                     flags=flags, stream=st)
    run = lambda name: _lib.check(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(descs[name])))
    ms = {n: [] for n in descs}
    out = {}
    for r in range(rounds):
        for name in (("off", "early_stop") if r % 2 == 0 else ("early_stop", "off")):
            for _ in range(3):
                run(name)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(steps):
                run(name)
            e1.record()
            torch.cuda.synchronize()
            ms[name].append(e0.elapsed_time(e1) / steps)
            out[name] = color.clone()
    run("early_stop")
    skipped, total = ctypes.c_ulonglong(), ctypes.c_ulonglong()
    _lib.check(lib.gmpi_debug_fwd_early_stop_stats(ctypes.byref(skipped), ctypes.byref(total)))
    assert int(flags.item()) == 0
    off, on = statistics.median(ms["off"]), statistics.median(ms["early_stop"])
    return {"ms_off": off, "ms_early_stop": on, "speedup": off / on, "ms_off_all": ms["off"], "ms_early_stop_all": ms["early_stop"],
            "stages_skipped_frac": skipped.value / max(total.value, 1),
            "max_abs_color_change": float((out["early_stop"] - out["off"]).abs().max())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tau", type=float, default=2.0 ** -24)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    dev = torch.device("cuda:0")
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"], capture_output=True,
                               text=True, timeout=30).stdout.strip()
    except Exception:
        power = "unknown"
    res = {"gpu": torch.cuda.get_device_name(dev), "power_limit": power, "tau": args.tau,
           "mpi": "synthetic (synth.make_head_case), not a trained GMPI MPI"}
    case = synth.make_head_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=1234, device=dev)
    res["headline_shape"] = dict(workload="96 planes, 1024^2, 4 MPIs x 1 view, forward",
                                 **measure(case, 1, args.tau, args.rounds, args.steps))
    del case
    yaws = np.linspace(0.5, -0.5, 120).astype(np.float32)
    case = synth.make_head_case(n_planes=96, tex=512, img=512, n_mpi=1, views_per_mpi=120, seed=1234, device=dev, yaws=yaws,
                                pitches=np.zeros(120, np.float32))
    res["video_512"] = dict(workload="96 planes, 512^2, 120 views of one MPI, forward",
                            **measure(case, 120, args.tau, args.rounds, args.steps))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
