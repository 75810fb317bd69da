"""CPU: every CUDA kernel of libgcbf_b200.so is defined in exactly one translation unit.  A kernel defined in a header is
compiled into every unit that includes it: the copies of a template kernel share one host stub, so the source does not
decide which copy a launch runs, and an inline launcher in a header names a different static kernel in each unit.
Headers under csrc/ therefore hold device functions, types, constants and stateless host helpers only; each kernel
lives in the .cu that owns its launcher."""
import collections
import os
import re
import shutil
import subprocess

import pytest

from helpers import ROOT

CSRC = os.path.join(ROOT, "gcbfplus_b200", "csrc")


def test_no_kernel_in_headers():
    offenders = []
    for fn in sorted(os.listdir(CSRC)):
        if fn.endswith(".cuh"):
            with open(os.path.join(CSRC, fn)) as f:
                if "__global__" in f.read():
                    offenders.append(fn)
    assert offenders == []


def test_build_units_are_the_cu_files():
    from gcbfplus_b200 import build
    assert set(build.UNITS) == {fn for fn in os.listdir(CSRC) if fn.endswith(".cu")}


def _cuobjdump():
    """cuobjdump of the CUDA toolkit whose nvcc builds the library (beside it), or the one on PATH."""
    from gcbfplus_b200 import build
    nvcc = build._nvcc()
    if os.path.isabs(nvcc):
        tool = os.path.join(os.path.dirname(nvcc), "cuobjdump")
        return tool if os.path.exists(tool) else None
    return shutil.which("cuobjdump")


def test_each_kernel_is_compiled_once():
    tool = _cuobjdump()
    if tool is None:
        pytest.skip("cuobjdump not found")
    from gcbfplus_b200 import _lib
    _lib.load()
    out = subprocess.run([tool, "-sass", _lib.lib_path()], capture_output=True, text=True, check=True).stdout
    names = re.findall(r"^\s*Function : (\S+)\s*$", out, flags=re.M)
    assert names, "no kernels found in the library"
    copies = {n: c for n, c in collections.Counter(names).items() if c > 1}
    assert copies == {}
