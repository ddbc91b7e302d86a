#!/usr/bin/env python
"""Train step (training forward + backward through autograd) with the default and the deterministic backward, alternating in one
process: median and min..max of CUDA-event times per configuration, plus the card and its power limit.

    python tools/deterministic_bench.py [--steps 10] [--warmup 3] [--out result.json]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import ml_gmpi_b200 as g  # noqa: E402
from ml_gmpi_b200 import synth  # noqa: E402

# (name, MPIs, views per MPI, planes, texture = image size, factored)
CONFIGS = [("4x1 view, 96 x 1024^2", 4, 1, 96, 1024, False),
           ("8x1 view, 32 x 256^2", 8, 1, 32, 256, False),
           ("4x1 view, 96 x 1024^2, factored + bg_rgb", 4, 1, 96, 1024, True)]


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run_config(name, M, vpm, N, T, factored, steps, warmup):
    d = torch.device("cuda:0")
    case = synth.make_case(n_planes=N, tex=T, img=T, n_mpi=M, views_per_mpi=vpm, seed=1, device=d, last_alpha_one=True)
    V = M * vpm
    gen = torch.Generator(device=d).manual_seed(2)
    gc = torch.randn((V, 3, T, T), generator=gen, device=d)
    gd = torch.randn((V, 1, T, T), generator=gen, device=d)
    if factored:
        mpi = [torch.rand((M, 3, T, T), generator=gen, device=d), torch.rand((M, N, 1, T, T), generator=gen, device=d),
               torch.rand((M, 3, T, T), generator=gen, device=d)]
        mpi[1][:, -1] = 1.0
        case.rgba = None
    else:
        mpi = [case.rgba]
    leaves = [t.requires_grad_(True) for t in mpi]

    def step(det):
        for t in leaves:
            t.grad = None
        if factored:
            color, depth = g.render_views_factored(leaves[0], leaves[1], case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir,
                                                   bg_rgb=leaves[2], view_group=vpm, deterministic=det)
        else:
            color, depth = g.render_views(leaves[0], case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, view_group=vpm,
                                          deterministic=det)
        ((color * gc).sum() + (depth * gd).sum()).backward()

    times = {False: [], True: []}
    for i in range(warmup + steps):
        for det in (False, True):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            torch.cuda.synchronize()
            a.record()
            step(det)
            b.record()
            torch.cuda.synchronize()
            if i >= warmup:
                times[det].append(a.elapsed_time(b))
    res = {"config": name}
    for det, key in ((False, "default"), (True, "deterministic")):
        t = times[det]
        res[key] = {"median_ms": round(statistics.median(t), 3), "min_ms": round(min(t), 3), "max_ms": round(max(t), 3)}
    res["ratio"] = round(res["deterministic"]["median_ms"] / res["default"]["median_ms"], 3)
    del leaves[:], mpi[:], case
    torch.cuda.empty_cache()
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "needs a CUDA device"
    out = {"card": card(), "results": [run_config(*c, a.steps, a.warmup) for c in CONFIGS]}
    for r in out["results"]:
        print(json.dumps(r))
    print("card:", out["card"])
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
