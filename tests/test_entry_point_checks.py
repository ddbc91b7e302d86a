"""What every render entry point answers for a matrix of descriptors: the option sets (none, fp16, uint8 and early stop, alone and
in pairs) crossed with the MPI form, a transmittance output, the camera and forward outputs or backward gradients, plus the previous
descriptor size, an out-of-range early_stop and view groups that do not divide V.  Each cell's return code, answer (size, plan and
reasons, kernel name) and refusal message must equal tests/golden/entry_point_codes.json.  The classic entry points get the same
cells, their arguments taken from the descriptor.

No call may reach a kernel.  Every descriptor but one variant has V = 0, so an accepted forward or backward returns before it
launches anything, and no cell sets GMPI_ZERO_GRAD.  The cells that would do GPU work if a call were accepted by mistake (the host
entry points and the occupancy build, which do GPU work whenever they accept a call, and every cell with V > 0) run only where CUDA
is not available, so that such a call fails with GMPI_ERR_CUDA instead of reading host pointers on a device.  The text of a
GMPI_ERR_CUDA message comes from the CUDA runtime, so only refusal messages are recorded.

    python tests/test_entry_point_checks.py --record   # rewrites tests/golden/entry_point_codes.json from the loaded library
"""
import ctypes
import itertools
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from ml_gmpi_b200 import _lib  # noqa: E402
from testlib import lib  # noqa: E402

RECORD = os.path.join(ROOT, "tests", "golden", "entry_point_codes.json")
F16, U8, ES = _lib.OPT_MPI_F16, _lib.OPT_MPI_U8, _lib.OPT_EARLY_STOP
OPTIONS = {"0": 0, "F16": F16, "U8": U8, "ES": ES, "F16|U8": F16 | U8, "F16|ES": F16 | ES, "U8|ES": U8 | ES}
MPIS = {"expanded": ("rgba",), "factored": ("rgb", "alpha"), "factored+bg": ("rgb", "alpha", "bg_rgb")}
IO = {"outputs": ("color", "depth", "flags"), "gradients": ("g_color", "g_depth")}
GRADS = {"rgba": "g_rgba", "rgb": "g_rgb", "alpha": "g_alpha", "bg_rgb": "g_bg_rgb"}
# the malformed variants; "plain" is crossed with every axis, the others with the options, MPI forms and outputs or gradients
VARIANTS = {"plain": {}, "v2_bytes": {"struct_bytes": _lib.RENDER_DESC_V2_BYTES}, "early_stop=1.5": {"early_stop": 1.5},
            "view_group=-1": {"view_group": -1}, "V=3,view_group=2": {"V": 3, "view_group": 2}}
BIG = 1 << 20          # the bytes of the host buffer every pointer of a cell points at (occupancy map and scratch included)


def descriptors():
    """[(name, fields)] of the matrix; the fields hold True for every pointer that is set."""
    out = []
    for var, extra in VARIANTS.items():
        plain = var == "plain"
        for opt, mpi, trans, cam, io in itertools.product(OPTIONS, MPIS, (False, True) if plain else (False,),
                                                          (False, True) if plain else (False,), IO):
            f = dict(M=1, V=0, N=2, Ht=8, Wt=8, H=8, W=8, options=OPTIONS[opt], early_stop=0.25, view2mpi=True, dhw=True)
            f.update({k: True for k in MPIS[mpi] + IO[io] + (("cam",) if cam else ("ray_dir", "eye", "z_dir"))})
            if io == "gradients":
                f.update({GRADS[k]: True for k in MPIS[mpi]})
            if trans:
                f["transmittance"] = True
            f.update(extra)
            out.append((f"{var} {opt} {mpi} {'transmittance' if trans else '-'} {'cam' if cam else 'rays'} {io}", f))
    return out


def make(fields, p):
    d = _lib.make_desc(**{k: (p if v is True else v) for k, v in fields.items() if k != "struct_bytes"})
    d.struct_bytes = fields.get("struct_bytes", d.struct_bytes)
    return d


def _int(rc):
    return rc, []


def _size(n):
    """A size query: the size, or a negative error code."""
    return (-n, []) if n < 0 else (0, [n])


def _plan(lib, call):
    why = ctypes.c_uint32(0)
    plan = call(ctypes.byref(why))
    return (-plan, []) if plan < 0 else (0, [plan, why.value])


def _classic(d):
    """The first six arguments of a classic entry point"""
    return [d.rgba, d.view2mpi, d.dhw, d.ray_dir, d.eye, d.z_dir]


def _sizes(d):
    return [d.M, d.V, d.N, d.Ht, d.Wt, d.H, d.W]


# {entry point: (does GPU work whenever it accepts a call, call(lib, desc, p) -> (GMPI_* code, answer))}
ENTRIES = {
    "fwd_ex": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_fwd_ex(ctypes.byref(d)))),
    "fwd_skip_ex": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_fwd_skip_ex(ctypes.byref(d), p, BIG))),
    "bwd_ex": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_bwd_ex(ctypes.byref(d)))),
    "bwd_deterministic_ex": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_bwd_deterministic_ex(ctypes.byref(d), p, BIG))),
    "bwd_deterministic_scratch_bytes": (False, lambda lib, d, p: _size(lib.gmpi_mpi_render_bwd_deterministic_scratch_bytes(ctypes.byref(d)))),
    "occupancy_bytes": (False, lambda lib, d, p: _size(lib.gmpi_mpi_occupancy_bytes(ctypes.byref(d)))),
    "fwd_plan_ex": (False, lambda lib, d, p: _plan(lib, lambda why: lib.gmpi_mpi_render_fwd_plan_ex(ctypes.byref(d), why))),
    "fwd": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_fwd(*_classic(d), d.color, d.depth, d.flags, *_sizes(d), d.options, None))),
    "fwd_train": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_fwd_train(*_classic(d), d.color, d.depth, d.transmittance, d.flags,
                                                                              *_sizes(d), d.options, None))),
    "fwd_gather": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_fwd_gather(*_classic(d), p, 1, 0, d.flags, *_sizes(d), d.options,
                                                                                None))),
    "bwd": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_bwd(*_classic(d), d.g_color, d.g_depth, d.g_rgba, *_sizes(d), d.options,
                                                                  None))),
    "bwd_saved": (False, lambda lib, d, p: _int(lib.gmpi_mpi_render_bwd_saved(*_classic(d), d.transmittance, d.g_color, d.g_depth,
                                                                              d.g_rgba, *_sizes(d), d.options, None))),
    "fwd_plan": (False, lambda lib, d, p: _plan(lib, lambda why: lib.gmpi_mpi_render_fwd_plan(d.V, d.N, d.Ht, d.Wt, d.H, d.W, d.rgba,
                                                                                              why))),
    "fwd_variant": (False, lambda lib, d, p: (0, [lib.gmpi_mpi_render_fwd_variant(d.N, d.Ht, d.Wt, d.H, d.W).decode()])),
    "host_ex": (True, lambda lib, d, p: _int(lib.gmpi_mpi_render_host_ex(ctypes.byref(d), 0))),
    "fwd_host": (True, lambda lib, d, p: _int(lib.gmpi_mpi_render_fwd_host(*_classic(d), d.color, d.depth, d.flags, *_sizes(d),
                                                                           d.options, 0))),
    "build_occupancy": (True, lambda lib, d, p: _int(lib.gmpi_mpi_build_occupancy(ctypes.byref(d), p, BIG))),
}


def run_cells(lib, with_gpu_work):
    """{entry point: {cell: [code, answer, message]}}; the message of a refusal (GMPI_ERR_INVALID_ARGUMENT or GMPI_ERR_UNSUPPORTED)
    only.  with_gpu_work: also the cells that would do GPU work if the call were accepted."""
    buf = (ctypes.c_char * (BIG + 256))()
    p = (ctypes.addressof(buf) + 255) & ~255
    out = {}
    for entry, (gpu_work, call) in ENTRIES.items():
        cells = out[entry] = {}
        for name, fields in descriptors():
            if (gpu_work or fields["V"] > 0) and not with_gpu_work:
                continue
            code, answer = call(lib, make(fields, p), p)
            cells[name] = [code, answer, lib.gmpi_last_error().decode() if code in (1, 3) else ""]
    return out


def load_record():
    """The record as run_cells returns it.  The file lists the cell names once, the distinct messages once, and per entry point
    [code, answer, message index] in the order of the names."""
    with open(RECORD) as f:
        r = json.load(f)
    return {e: {n: [c, a, r["messages"][m]] for n, (c, a, m) in zip(r["cells"], rows)} for e, rows in r["entry_points"].items()}


def write_record(cells):
    names = [n for n, _ in descriptors()]
    messages = sorted({m for c in cells.values() for _, _, m in c.values()})
    rows = {e: [[*c[n][:2], messages.index(c[n][2])] for n in names] for e, c in cells.items()}
    with open(RECORD, "w") as f:
        f.write('{"cells": ' + json.dumps(names, indent=0) + ',\n"messages": ' + json.dumps(messages, indent=0) + ',\n"entry_points": {\n' +
                ",\n".join(f"{json.dumps(e)}: {json.dumps(r, separators=(',', ':'))}" for e, r in rows.items()) + "\n}}\n")


def test_every_entry_point_answers_every_cell_as_recorded(lib):
    rec = load_record()
    got = run_cells(lib, with_gpu_work=not torch.cuda.is_available())
    diffs = []
    for entry, cells in got.items():
        assert entry in rec, entry
        for name, (code, answer, msg) in cells.items():
            r_code, r_answer, r_msg = rec[entry][name]
            if [code, answer, msg] != [r_code, r_answer, r_msg]:
                diffs.append(f"{entry} [{name}]: {code} {answer} {msg!r}, recorded {r_code} {r_answer} {r_msg!r}")
    assert not diffs, f"{len(diffs)} cells differ:\n" + "\n".join(diffs[:50])
    if not torch.cuda.is_available():
        assert {e: set(c) for e, c in got.items()} == {e: set(c) for e, c in rec.items()}


def test_the_matrix_reaches_every_kind_of_answer(lib):
    """The matrix is not all refusals: every entry point accepts some cell, and the descriptor entry points refuse with both codes."""
    for entry, cells in load_record().items():
        codes = {c[0] for c in cells.values()}
        assert codes & {0, 2}, entry                  # accepted (GMPI_ERR_CUDA: accepted, then no device)
        if entry not in ("fwd_plan", "fwd_variant", "fwd_plan_ex"):
            assert {1, 3} <= codes, entry


if __name__ == "__main__" and "--record" in sys.argv:
    assert not torch.cuda.is_available(), "record where CUDA is not available, so that every cell is called"
    cells = run_cells(_lib.load(), with_gpu_work=True)
    write_record(cells)
    print("wrote", RECORD, sum(len(c) for c in cells.values()), "cells")
