#!/usr/bin/env python
"""Forward time of fp32 against 8-bit MPIs (GMPI_MPI_U8):
    python tools/unorm8_bench.py [--rounds 5] [--steps 10] [--out result.json]
Workloads: 4 MPIs x 1 view, 96 planes, 1024^2 (bench.py's headline shape), expanded; the 512^2 video sweep (120 views of one
96-plane MPI, uint8 frames, views grouped); the host entry point (gmpi_mpi_render_host_ex) on 2 MPIs x 2 views, 96 planes, 512^2
from pinned host buffers, where the upload dominates.  Per workload three forms alternate within every round: fp32 (the fp32 MPI
the codes stand for), u8 (native), and upcast (what a uint8 MPI cost before: the exact conversion unorm8_to_float, then the fp32
render).  Prints the medians over the rounds and their spread (min..max), and checks that the u8 and fp32 outputs are bitwise
equal.  The card's name and power limit are read in the same run."""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import ml_gmpi_b200 as g
from ml_gmpi_b200 import _lib, synth


def timed(fn, steps):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def compare(forms, rounds, steps):
    """forms: name -> callable; alternated (rotated) within each round.  Returns {name: {median_ms, min_ms, max_ms}}."""
    ms = {n: [] for n in forms}
    names = list(forms)
    for r in range(rounds):
        for n in names[r % len(names):] + names[:r % len(names)]:
            ms[n].append(timed(forms[n], steps))
    return {n: dict(median_ms=round(statistics.median(v), 4), min_ms=round(min(v), 4), max_ms=round(max(v), 4)) for n, v in ms.items()}


def quantize(x):
    return (x * 255.0).round_().clamp_(0, 255).to(torch.uint8)


def device_forms(case, video, view_group):
    u8 = quantize(case.rgba)
    f32 = g.unorm8_to_float(u8)
    vid = {"near": 0.88, "far": 1.12} if video else None
    kw = dict(dhw=case.dhw, view2mpi=case.view2mpi, ray_dir=case.ray_dir, eye=case.eye, z_dir=case.z_dir, view_group=view_group, video=vid)

    def render(x, unorm8=False):
        with torch.no_grad():
            return g.render_frames(rgba=x, unorm8=unorm8, **kw)

    forms = {"fp32": lambda: render(f32), "u8": lambda: render(u8, True), "upcast": lambda: render(g.unorm8_to_float(u8))}
    same = all(torch.equal(a, b) for a, b in zip(render(u8, True), render(f32)))
    return forms, same


def host_forms(case):
    lib = _lib.load()
    V, _, H, W = case.ray_dir.shape
    M, N, _, Ht, Wt = case.rgba.shape
    pin = lambda t: t.contiguous().pin_memory()
    x8 = pin(quantize(case.rgba))
    x32 = pin(g.unorm8_to_float(x8))
    inputs = {k: pin(getattr(case, k)) for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
    color, depth = pin(torch.empty((V, 3, H, W))), pin(torch.empty((V, 1, H, W)))
    flags = torch.zeros(1, dtype=torch.int32)

    def run(x, u8):
        d = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | (_lib.OPT_MPI_U8 if u8 else 0), M=M, V=V,
                           N=N, Ht=Ht, Wt=Wt, H=H, W=W, rgba=x, color=color, depth=depth, flags=flags, **inputs)
        _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0))
        return color.clone(), depth.clone()

    same = all(torch.equal(a, b) for a, b in zip(run(x8, True), run(x32, False)))
    return {"fp32": lambda: run(x32, False), "u8": lambda: run(x8, True), "upcast": lambda: run(g.unorm8_to_float(x8), False)}, same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "unorm8_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    res = {"gpu": smi[0] if smi else "unknown", "rounds": a.rounds, "steps": a.steps, "workloads": {}, "bitwise_equal": {}}
    rand = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=3, last_alpha_one=True, device=dev)
    forms, res["bitwise_equal"]["4x96x1024_expanded"] = device_forms(rand, False, 1)
    res["workloads"]["4x96x1024_expanded"] = compare(forms, a.rounds, a.steps)
    del rand, forms
    torch.cuda.empty_cache()
    sweep = synth.make_case(n_planes=96, tex=512, img=512, n_mpi=1, views_per_mpi=120, seed=5, last_alpha_one=True, device=dev)
    forms, res["bitwise_equal"]["video_120x512"] = device_forms(sweep, True, 120)
    res["workloads"]["video_120x512"] = compare(forms, a.rounds, a.steps)
    del sweep, forms
    torch.cuda.empty_cache()
    hcase = synth.make_case(n_planes=96, tex=512, img=512, n_mpi=2, views_per_mpi=2, seed=6, last_alpha_one=True)
    forms, res["bitwise_equal"]["host_2x96x512"] = host_forms(hcase)
    res["workloads"]["host_2x96x512"] = compare(forms, a.rounds, max(1, a.steps // 5))
    for w in res["workloads"].values():
        w["u8_speedup"] = round(w["fp32"]["median_ms"] / w["u8"]["median_ms"], 3)
        w["u8_vs_upcast"] = round(w["upcast"]["median_ms"] / w["u8"]["median_ms"], 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
