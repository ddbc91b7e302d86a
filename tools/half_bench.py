#!/usr/bin/env python
"""Forward time of fp32 against fp16 MPIs (GMPI_MPI_F16):
    python tools/half_bench.py [--rounds 5] [--steps 10] [--out result.json]
Workloads: 4 MPIs x 1 view, 96 planes, 1024^2 (bench.py's headline shape), expanded and factored; the 512^2 video sweep (120
views of one 96-plane MPI, uint8 frames, views grouped); the host entry point (gmpi_mpi_render_host_ex) on 2 MPIs x 2 views,
96 planes, 512^2 from pinned host buffers, where the upload dominates.  Per workload three forms alternate within every round:
fp32 (the fp32 MPI), fp16 (native), and upcast (what an fp16 MPI cost before: .float() then the fp32 render).  Prints the
medians over the rounds and their spread (min..max), and the largest colour difference between the fp16 render and the fp32
render of the ORIGINAL fp32 MPI (what quantising the MPI costs) on random inputs and on synth.make_head_case.  The card's name
and power limit are read in the same run."""
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


def device_forms(case, factored, video, view_group):
    x32 = case.rgba
    if factored:
        mpi32 = dict(rgb=x32[:, 0, :3].contiguous(), alpha=x32[:, :, 3:4].contiguous())
    else:
        mpi32 = dict(rgba=x32)
    mpi16 = {k: v.half() for k, v in mpi32.items()}
    vid = {"near": 0.88, "far": 1.12} if video else None
    kw = dict(dhw=case.dhw, view2mpi=case.view2mpi, ray_dir=case.ray_dir, eye=case.eye, z_dir=case.z_dir, view_group=view_group, video=vid)

    def render(mpi):
        with torch.no_grad():
            return g.render_frames(**kw, **mpi)

    forms = {"fp32": lambda: render(mpi32), "fp16": lambda: render(mpi16),
             "upcast": lambda: render({k: v.float() for k, v in mpi16.items()})}
    return forms, (lambda m: render(m)), mpi32, mpi16


def quant_error(render, mpi32, mpi16):
    """largest colour difference, in [0, 1] colour units (uint8 codes / 255, or colour in [-1, 1] / 2)"""
    a, b = render(mpi32)[0], render(mpi16)[0]
    return float((a.float() - b.float()).abs().max()) / (255.0 if a.dtype == torch.uint8 else 2.0)


def host_forms(case):
    lib = _lib.load()
    V, _, H, W = case.ray_dir.shape
    M, N, _, Ht, Wt = case.rgba.shape
    pin = lambda t: t.contiguous().pin_memory()
    x32 = pin(case.rgba)
    x16 = pin(case.rgba.half())
    inputs = {k: pin(getattr(case, k)) for k in ("view2mpi", "dhw", "ray_dir", "eye", "z_dir")}
    color, depth = pin(torch.empty((V, 3, H, W))), pin(torch.empty((V, 1, H, W)))
    flags = torch.zeros(1, dtype=torch.int32)

    def run(x, f16):
        d = _lib.make_desc(options=_lib.OPT_ALIGN_CORNERS | _lib.OPT_COLOR_MINUS1_1 | (_lib.OPT_MPI_F16 if f16 else 0), M=M, V=V,
                           N=N, Ht=Ht, Wt=Wt, H=H, W=W, rgba=x, color=color, depth=depth, flags=flags, **inputs)
        _lib.check(lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0))

    return {"fp32": lambda: run(x32, False), "fp16": lambda: run(x16, True),
            "upcast": lambda: run(x16.float(), False)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "half_bench measures on a CUDA device"
    dev = torch.device("cuda:0")
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip().splitlines()
    res = {"gpu": smi[0] if smi else "unknown", "rounds": a.rounds, "steps": a.steps, "workloads": {}, "quantisation": {}}
    rand = synth.make_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=3, last_alpha_one=True, device=dev)
    for name, factored in (("4x96x1024_expanded", False), ("4x96x1024_factored", True)):
        forms, render, m32, m16 = device_forms(rand, factored, False, 1)
        res["workloads"][name] = compare(forms, a.rounds, a.steps)
        res["quantisation"][name + "_random"] = quant_error(render, m32, m16)
        del forms, render, m32, m16
    del rand
    torch.cuda.empty_cache()
    hc = synth.make_head_case(n_planes=96, tex=1024, img=1024, n_mpi=4, seed=4, device=dev)
    _, render, m32, m16 = device_forms(hc, False, False, 1)
    res["quantisation"]["4x96x1024_head_case"] = quant_error(render, m32, m16)
    del hc, render, m32, m16
    torch.cuda.empty_cache()
    sweep = synth.make_case(n_planes=96, tex=512, img=512, n_mpi=1, views_per_mpi=120, seed=5, last_alpha_one=True, device=dev)
    forms, render, m32, m16 = device_forms(sweep, False, True, 120)
    res["workloads"]["video_120x512"] = compare(forms, a.rounds, a.steps)
    res["quantisation"]["video_120x512_random_u8"] = quant_error(render, m32, m16)
    del sweep, forms, render, m32, m16
    torch.cuda.empty_cache()
    hcase = synth.make_case(n_planes=96, tex=512, img=512, n_mpi=2, views_per_mpi=2, seed=6, last_alpha_one=True)
    res["workloads"]["host_2x96x512"] = compare(host_forms(hcase), a.rounds, max(1, a.steps // 5))
    for w in res["workloads"].values():
        w["fp16_speedup"] = round(w["fp32"]["median_ms"] / w["fp16"]["median_ms"], 3)
        w["fp16_vs_upcast"] = round(w["upcast"]["median_ms"] / w["fp16"]["median_ms"], 3)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
