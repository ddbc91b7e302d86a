"""CPU checks of the built library: one artifact holds every kernel, the skipping (mpi_skip.cu) and uint8 (mpi_u8.cu) ones included,
and every kernel keeps the machine code recorded in tests/golden/sass_digests.json (testlib.library_kernels reads the machine code).

    python tests/test_library_build.py --record-sass   # rewrites tests/golden/sass_digests.json
"""
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
from testlib import KEY_U8, library_kernels, render_kernels  # noqa: E402

SASS_DIGESTS = os.path.join(ROOT, "tests", "golden", "sass_digests.json")


def _nvcc_release():
    out = subprocess.run([g._build.nvcc_path(), "--version"], capture_output=True, text=True).stdout
    m = re.search(r"release [0-9.]+, V[0-9.]+", out)
    return m.group(0) if m else out.strip()


def test_sass_of_every_kernel_is_recorded_by_template_and_key():
    """Every kernel of the library has the recorded machine code, instruction for instruction: none changed, none missing, none
    unrecorded (the record names the compiler release it was taken with)."""
    with open(SASS_DIGESTS) as f:
        rec = json.load(f)
    if _nvcc_release() != rec["nvcc"]:
        pytest.skip(f"machine code recorded with nvcc {rec['nvcc']}, this is {_nvcc_release()}")
    g.build_library()
    assert {n: k.digest() for n, k in library_kernels().items()} == rec["kernels"]


def test_clean_build_makes_one_library_with_every_kernel_key(tmp_path):
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
    kernels = library_kernels(lib)
    skip = set(render_kernels(kernels, "mpi_fwd_skip_kernel", lacks=KEY_U8)) | {n for n in kernels if re.fullmatch(r"gmpi_occ_\w+_f(32|16)", n)}
    u8 = {n for n, k in kernels.items() if k.key is not None and k.key & KEY_U8}
    assert len(skip) == 20 and len(u8) == 12 and {"gmpi_occ_expanded_u8", "gmpi_u8_codes"} <= set(kernels), sorted(kernels)


if __name__ == "__main__" and "--record-sass" in sys.argv:
    g.build_library()
    with open(SASS_DIGESTS, "w") as f:
        json.dump({"nvcc": _nvcc_release(), "kernels": {n: k.digest() for n, k in library_kernels().items()}}, f, indent=1,
                  sort_keys=True)
        f.write("\n")
    print("wrote", SASS_DIGESTS)
