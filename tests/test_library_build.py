"""CPU checks of the built library: one artifact holds every kernel, the skipping (mpi_skip.cu) and uint8 (mpi_u8.cu) ones included,
and every kernel keeps the machine code recorded in tests/golden/sass_digests.json.  library_kernels() reads a built library's kernels
for the machine-code tests of the other modules too.

    python tests/test_library_build.py --record-sass   # rewrites tests/golden/sass_digests.json
"""
import hashlib
import json
import os
import re
import shutil
import subprocess
import sys
from typing import NamedTuple, Optional

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


# The render-kernel key bits (kKey*, csrc/mpi_kernel_keys.cuh)
KEY_AC, KEY_FAC, KEY_EMIT, KEY_ES, KEY_F16, KEY_STAGED, KEY_BWD, KEY_DET, KEY_SKIP, KEY_U8 = 1, 2, 4, 8, 16, 32, 64, 128, 256, 512


class Kernel(NamedTuple):
    template: str           # the C++ name: a kernel template, or a plain or extern "C" kernel
    key: Optional[int]      # the render kernel's key (template<uint32_t K>), None for other kernels
    sass: str
    regs: int
    stack: int
    local: int

    def digest(self):
        """sha256 of the SASS instructions (addresses and encodings included, no names or comments)"""
        lines = [l.strip() for l in self.sass.split("\n") if re.match(r"\s+/\*[0-9a-f]{4,}\*/", l)]
        return hashlib.sha256("\n".join(lines).encode()).hexdigest()


def library_kernels(path=None):
    """{mangled name: Kernel} of a built library (cuobjdump -sass and -res-usage).  Kernels of namespace gmpi are
    _ZN4gmpi<length><name>..., and a uint32_t template argument K mangles as ILj<K>E."""
    path = path or g._build.LIB_PATH
    run = lambda flag: subprocess.run(["cuobjdump", flag, path], capture_output=True, text=True, check=True).stdout
    usage = {m[1]: (int(m[2]), int(m[3]), int(m[4]))
             for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", run("-res-usage"))}
    out = {}
    for f in re.split(r"\n\s*Function : ", run("-sass"))[1:]:
        name, body = f.split("\n", 1)
        name = name.strip()
        template, key = name, None
        m = re.match(r"_ZN4gmpi(\d+)", name)
        if m:
            end = m.end() + int(m[1])
            template = name[m.end():end]
            k = re.match(r"ILj(\d+)EE", name[end:])
            key = int(k[1]) if k else None
        out[name] = Kernel(template, key, body, *usage[name])
    return out


def render_kernels(kernels, template, has=0, lacks=0):
    """{name: Kernel} of the instantiations of `template` whose key has every bit of `has` and none of `lacks`"""
    return {n: k for n, k in kernels.items() if k.template == template and k.key & has == has and not k.key & lacks}


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
