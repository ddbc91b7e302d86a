"""CPU checks of the built library: one artifact holds every kernel, the skipping (mpi_skip.cu) and uint8 (mpi_u8.cu) ones included,
and every kernel keeps the machine code recorded in tests/golden/sass_digests.json.

    python tests/test_library_build.py --record-sass   # rewrites tests/golden/sass_digests.json
"""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import ml_gmpi_b200 as g  # noqa: E402

SASS_DIGESTS = os.path.join(ROOT, "tests", "golden", "sass_digests.json")


def _nvcc_release():
    out = subprocess.run([g._build.nvcc_path(), "--version"], capture_output=True, text=True).stdout
    m = re.search(r"release [0-9.]+, V[0-9.]+", out)
    return m.group(0) if m else out.strip()


def sass_digests(path):
    """{mangled kernel name: sha256 of its SASS instructions} of a built library (cuobjdump -sass)."""
    txt = subprocess.run(["cuobjdump", "-sass", path], capture_output=True, text=True, check=True).stdout
    out = {}
    for f in re.split(r"\n\s*Function : ", txt)[1:]:
        name, body = f.split("\n", 1)
        lines = [l.strip() for l in body.split("\n") if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
        out[name.strip()] = hashlib.sha256("\n".join(lines).encode()).hexdigest()
    return out


def test_sass_of_every_kernel_is_recorded():
    """Every kernel of the library has the recorded machine code, instruction for instruction: none changed, none missing, none
    unrecorded (the record names the compiler release it was taken with)."""
    with open(SASS_DIGESTS) as f:
        rec = json.load(f)
    if _nvcc_release() != rec["nvcc"]:
        pytest.skip(f"machine code recorded with nvcc {rec['nvcc']}, this is {_nvcc_release()}")
    g.build_library()
    assert sass_digests(g._build.LIB_PATH) == rec["kernels"]


def test_clean_build_makes_one_library_with_every_kernel(tmp_path):
    """A clean build of a copy of the sources writes the library and nothing else (no kernel module beside it), and the library
    holds the skipping and uint8 kernels."""
    pkg = tmp_path / "ml_gmpi_b200"
    shutil.copytree(g._build.CSRC, pkg / "csrc")
    shutil.copytree(os.path.join(ROOT, "include"), tmp_path / "include")
    shutil.copy(g._build.__file__, pkg / "_build.py")
    before = set(os.listdir(pkg))
    code = "import _build; print(_build.build_library(force=True))"
    res = subprocess.run([sys.executable, "-B", "-c", code], cwd=pkg, capture_output=True, text=True)
    assert res.returncode == 0, res.stdout + res.stderr
    lib = str(pkg / "libgmpi_mpi_render.so")
    assert res.stdout.strip() == lib
    assert set(os.listdir(pkg)) - before == {"libgmpi_mpi_render.so"}
    assert not [f for f in os.listdir(pkg) if f.endswith(".fatbin")]
    kernels = set(sass_digests(lib))
    skip = {n for n in kernels if n.startswith("gmpi_fwd_skip_")} | {n for n in kernels if re.fullmatch(r"gmpi_occ_\w+_f(32|16)", n)}
    u8 = {n for n in kernels if re.fullmatch(r"gmpi_(fwd_u8_(skip_)?|fwd_direct_u8_)a[01]_e[01]", n)}
    assert len(skip) == 20 and len(u8) == 12 and {"gmpi_occ_expanded_u8", "gmpi_u8_codes"} <= kernels, sorted(kernels)


if __name__ == "__main__" and "--record-sass" in sys.argv:
    g.build_library()
    with open(SASS_DIGESTS, "w") as f:
        json.dump({"nvcc": _nvcc_release(), "kernels": sass_digests(g._build.LIB_PATH)}, f, indent=1, sort_keys=True)
        f.write("\n")
    print("wrote", SASS_DIGESTS)
