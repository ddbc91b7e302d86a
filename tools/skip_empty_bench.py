#!/usr/bin/env python
"""Forward render with empty-space skipping off and on (render_frames(skip_empty=...)), alternating in one process, 5 rounds: median
and min..max of CUDA-event times per configuration, the occupancy-map build on its own, the skipped-stage fraction, and the card
and its power limit.  "on" reuses a map built once per MPI; "build" is that map's build time.

    python tools/skip_empty_bench.py [--rounds 5] [--reps 5] [--out result.json]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ml_gmpi_b200 as g  # noqa: E402
from ml_gmpi_b200 import _lib, service, synth  # noqa: E402
from ml_gmpi_b200.camera import PinholeCamera  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def workloads(d):
    """(name, MPI kwargs, ray kwargs, view_group) of each workload, on device d."""
    head = synth.make_head_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=1, device=d)
    rays = dict(ray_dir=head.ray_dir, eye=head.eye, z_dir=head.z_dir, dhw=head.dhw, view2mpi=head.view2mpi)
    gen = torch.Generator(device=d).manual_seed(3)
    rgb = torch.rand((4, 3, 1024, 1024), generator=gen, device=d)
    out = [("head 4 x 96 x 1024^2, expanded", dict(rgba=head.rgba), rays, 1),
           ("head 4 x 96 x 1024^2, factored", dict(rgb=rgb, alpha=head.rgba[:, :, 3:4].contiguous()), rays, 1),
           ("head 4 x 96 x 1024^2, fp16", dict(rgba=head.rgba.half()), rays, 1)]
    rnd = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=2, device=d, last_alpha_one=True)
    out.append(("random 4 x 96 x 1024^2 (nothing empty)", dict(rgba=rnd.rgba), dict(ray_dir=rnd.ray_dir, eye=rnd.eye, z_dir=rnd.z_dir,
                                                                                      dhw=rnd.dhw, view2mpi=rnd.view2mpi), 1))
    # the video sweep: 120 views of one head MPI at 512^2.  From a 1024^2 texture a 64-pixel tile spans about 128 texels, more than the
    # widest staged box: every stage takes the generic body, which is never skipped.  A 512^2 texture stages every box.
    c2w = service.sphere_poses(torch.linspace(-0.3, 0.3, 120).reshape(-1, 1), torch.zeros(120, 1), (0.0, 0.0, 1.0), 1.0)
    ray_dir, eye, z_dir = PinholeCamera.from_fov(12.6, 512, 512).generate_rays(c2w.to(d))
    for tex in (512, 1024):
        one = synth.make_head_case(n_planes=96, tex=tex, img=512, n_mpi=1, seed=4, device=d)
        out.append((f"sweep 120 views of 96 x {tex}^2 at 512^2", dict(rgba=one.rgba),
                    dict(ray_dir=ray_dir, eye=eye, z_dir=z_dir, dhw=one.dhw, view2mpi=torch.zeros(120, dtype=torch.int32, device=d)), 120))
    return out


def timed(fn, reps):
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    torch.cuda.synchronize()
    return s.elapsed_time(e) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    d = torch.device("cuda:0")
    lib = _lib.load()
    res = {"card": card(), "rounds": a.rounds, "reps": a.reps, "results": []}
    with torch.no_grad():
        for name, mpi, rays, vg in workloads(d):
            for tau in (None, 0.01):
                occ = g.build_occupancy(**mpi)
                run = lambda skip: g.render_frames(**mpi, **rays, view_group=vg, early_stop=tau, skip_empty=occ if skip else False)
                run(False), run(True), g.build_occupancy(**mpi)         # warm-up: module loads, shapes
                t = {"off": [], "on": [], "build": []}
                for _ in range(a.rounds):
                    t["off"].append(timed(lambda: run(False), a.reps))
                    t["on"].append(timed(lambda: run(True), a.reps))
                    t["build"].append(timed(lambda: g.build_occupancy(**mpi), a.reps))
                run(True)
                s, tot = ctypes.c_ulonglong(0), ctypes.c_ulonglong(0)
                _lib.check(lib.gmpi_debug_fwd_skip_stats(ctypes.byref(s), ctypes.byref(tot)))
                row = {"workload": name, "early_stop": tau, "skipped_stage_fraction": s.value / tot.value if tot.value else 0.0}
                for k, v in t.items():
                    row[k + "_ms"] = {"median": statistics.median(v), "min": min(v), "max": max(v)}
                row["on_over_off"] = row["on_ms"]["median"] / row["off_ms"]["median"]
                res["results"].append(row)
                print(f"{name:45s} es={tau!s:5s} off {row['off_ms']['median']:8.3f} ms  on {row['on_ms']['median']:8.3f} ms "
                      f"({min(t['on']):.3f}..{max(t['on']):.3f})  build {row['build_ms']['median']:7.3f} ms  "
                      f"on/off {row['on_over_off']:.3f}  skipped {row['skipped_stage_fraction']:.3f}", flush=True)
    print(res["card"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
