"""In-tree build of libgcbf_b200.so with nvcc for sm_90a (H100; no torch dependency).

``python -m gcbfplus_b200.build`` or ``gcbfplus_b200.build.build()``.  The shared library
lands in gcbfplus_b200/lib/ (git-ignored build product).
All CUDA units are compiled with -fmad=false (bit-exact index / mask work, one numeric path; see DESIGN.md).
"""
from __future__ import annotations

import hashlib
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
LIBDIR = os.path.join(HERE, "lib")
LIB = os.path.join(LIBDIR, "libgcbf_b200.so")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xcompiler", "-fvisibility=hidden"]
# Every unit is compiled with -fmad=false: geometry.cu / rollout_persist.cu need one rounding per operation for the
# bit-exact LiDAR / index / mask work, and the others share device functions with them (edge features: sinf / cosf of
# the DubinsCar heading are inlined under the translation unit's contraction setting, so mixed settings made the
# persistent kernel and the 5-launch path differ in the last bit).  The GEMM-side hot loops use explicit fmaf.
UNITS = {  # translation unit -> extra flags
    "api.cu": [],
    "cbfqp.cu": ["-fmad=false"],
    "geometry.cu": ["-fmad=false"],
    "gnn.cu": ["-fmad=false"],
    "rollout_persist.cu": ["-fmad=false"],
    "train.cu": ["-fmad=false"],
}


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", "nvcc"):
        if c and (os.path.isabs(c) and os.path.exists(c) or not os.path.isabs(c)):
            return c
    return "nvcc"


def _digest() -> str:
    h = hashlib.sha256()
    for root in (CSRC, os.path.join(HERE, "..", "include")):
        for fn in sorted(os.listdir(root)):
            if fn.endswith((".cu", ".cuh", ".h")):
                with open(os.path.join(root, fn), "rb") as f:
                    h.update(fn.encode())
                    h.update(f.read())
    return h.hexdigest()


LAST = {"compiled": 0, "reused": 0}   # what the last build() call did (printed by __graft_entry__.build)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(LIBDIR, exist_ok=True)
    stamp = os.path.join(LIBDIR, "build.stamp")
    dig = _digest()
    n_units = sum(os.path.exists(os.path.join(CSRC, u)) for u in UNITS)
    if not force and os.path.exists(LIB) and os.path.exists(stamp) and open(stamp).read().strip() == dig:
        LAST.update(compiled=0, reused=n_units)
        return LIB
    nvcc = _nvcc()
    objs = []
    procs = []
    for unit, extra in UNITS.items():
        src = os.path.join(CSRC, unit)
        if not os.path.exists(src):
            continue
        obj = os.path.join(LIBDIR, unit.replace(".cu", ".o"))
        cmd = [nvcc, *ARCH, *COMMON, *extra, "-c", src, "-o", obj]
        if verbose:
            print(" ".join(cmd), file=sys.stderr)
        procs.append((unit, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        objs.append(obj)
    for unit, p in procs:
        out, _ = p.communicate()
        if p.returncode != 0:
            raise RuntimeError(f"nvcc failed on {unit}:\n{out.decode()}")
        if verbose and out:
            print(out.decode(), file=sys.stderr)
    cmd = [nvcc, *ARCH, "-shared", "-o", LIB, *objs, "-lcudart"]
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)
    if r.returncode != 0:
        raise RuntimeError(f"link failed:\n{r.stdout.decode()}")
    with open(stamp, "w") as f:
        f.write(dig)
    LAST.update(compiled=len(objs), reused=0)
    return LIB


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose=True))
