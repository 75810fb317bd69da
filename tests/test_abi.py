"""CPU: the C-ABI library loads and exports every symbol include/gcbf_b200.h declares
(no compute calls without a GPU), and host-side layout queries agree with Python."""
import ctypes
import os
import re

from helpers import ROOT

HEADER = os.path.join(ROOT, "include", "gcbf_b200.h")


def _declared_symbols():
    src = open(HEADER).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(gcbf_[a-z0-9_]+)\s*\(", src)))


def test_every_declared_symbol_is_exported():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    names = _declared_symbols()
    assert len(names) >= 10
    for n in names:
        assert hasattr(lib, n), f"{n} declared in gcbf_b200.h but not exported"


def test_every_exported_symbol_is_declared():
    import subprocess
    from gcbfplus_b200 import _lib
    _lib.load()
    out = subprocess.run(["nm", "-D", "--defined-only", _lib.lib_path()], capture_output=True, text=True).stdout
    exported = sorted(set(re.findall(r" T (gcbf_[a-z0-9_]+)", out)))
    assert exported == _declared_symbols()


def test_param_layout_matches_reference_counts():
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo.params import layer_specs
    # SURVEY A.3 parameter counts of the pretrained pickles
    for ed, nu, want_cbf, want_actor in [(2, 2, 365698, 365955), (4, 2, 366210, 366467), (6, 3, 366722, 367236)]:
        assert sum(i * o + o for _, i, o in layer_specs(ed, 1, "cbf")) == want_cbf
        assert sum(i * o + o for _, i, o in layer_specs(ed, nu, "actor")) == want_actor
        offs = _lib.param_offsets(ed, nu)
        assert all(o % 4 == 0 for o in offs) and offs == sorted(offs)
        assert _lib.param_count(ed, nu) >= want_actor


def test_layout_query_and_graph_build_report_errors_without_gpu():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    assert lib.gcbf_version() >= 100
    rc = lib.gcbf_param_offsets_l(99, 1, 1, (ctypes.c_int32 * 24)())
    assert rc < 0 and b"bad argument" in lib.gcbf_last_error_string()
    d = _lib.EnvDesc()
    d.env_kind = 7
    rc = lib.gcbf_graph_build(ctypes.byref(d), None, None, None, None, None, None, None, None, None, 1, None)
    assert rc < 0 and lib.gcbf_last_error_string()


def test_desc_struct_size_matches_header():
    from gcbfplus_b200 import _lib
    # 8 int32 + 21 float + K[18] + A[36] + B[18]
    assert ctypes.sizeof(_lib.EnvDesc) == 4 * (8 + 21 + 18 + 36 + 18)


def test_sqrt_threshold_is_exact():
    import numpy as np
    from gcbfplus_b200 import _lib
    for r in (0.5, 0.4, 0.1, 0.15000000000000002):
        a = np.float32(_lib.sqrt_threshold(r))
        r32 = np.float32(r)
        below = np.nextafter(a, np.float32(0), dtype=np.float32)
        assert np.sqrt(a) >= r32 and np.sqrt(below) < r32
        xs = np.linspace(float(a) * 0.999, float(a) * 1.001, 20001).astype(np.float32)
        assert np.array_equal(np.sqrt(xs) < r32, xs < a)
