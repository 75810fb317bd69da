"""ctypes binding of libgcbf_b200.so (the C ABI in include/gcbf_b200.h).

The product path has NO fallback: if the shared library is missing and cannot be
built, or a call returns a non-zero status, a RuntimeError is raised.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, "lib", "libgcbf_b200.so")

ENV_KIND = {"SingleIntegrator": 0, "DoubleIntegrator": 1, "DubinsCar": 2, "LinearDrone": 3}
NET_CBF, NET_ACTOR = 0, 1


class EnvDesc(C.Structure):
    """Mirror of `gcbf_env_desc` (include/gcbf_b200.h)."""
    _fields_ = [
        ("env_kind", C.c_int32), ("n_graphs", C.c_int32), ("n_agents", C.c_int32), ("n_obs", C.c_int32),
        ("n_rays", C.c_int32), ("n_hits", C.c_int32), ("edge_cap", C.c_int32), ("obs_per_graph", C.c_int32),
        ("comm_radius", C.c_float), ("comm_radius_p1", C.c_float), ("lidar_radius", C.c_float),
        ("dt", C.c_float), ("mass", C.c_float), ("radius", C.c_float), ("two_r", C.c_float),
        ("two_r_p1", C.c_float), ("half_r", C.c_float), ("unsafe_agent", C.c_float), ("unsafe_obs", C.c_float),
        ("warn_agent", C.c_float), ("warn_obs", C.c_float), ("four_r_sq", C.c_float), ("r_sq", C.c_float),
        ("safe_agent", C.c_float), ("safe_obs", C.c_float), ("comm_sq_thr", C.c_float), ("lidar_sq_thr", C.c_float),
        ("v_lim", C.c_float), ("u_lim", C.c_float),
        ("K", C.c_float * 18), ("A", C.c_float * 36), ("B", C.c_float * 18),
    ]

    def copy(self) -> "EnvDesc":
        out = EnvDesc()
        C.memmove(C.byref(out), C.byref(self), C.sizeof(EnvDesc))
        return out


_lib: Optional[C.CDLL] = None

_P = C.c_void_p
_SIGNATURES = {
    "gcbf_last_error_string": (C.c_char_p, []),
    "gcbf_version": (C.c_int32, []),
    "gcbf_launch_count": (C.c_int64, []),
    "gcbf_param_count_l": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32]),
    "gcbf_param_offsets_l": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(C.c_int32)]),
    "gcbf_graph_build": (C.c_int32, [C.POINTER(EnvDesc)] + [_P] * 9 + [C.c_int32, _P]),
    "gcbf_gnn_workspace_floats_l": (C.c_int64, [C.POINTER(EnvDesc), C.c_int32, C.c_int32]),
    "gcbf_gnn_forward_l": (C.c_int32, [C.POINTER(EnvDesc), C.c_int32, C.c_int32, C.c_int32] + [_P] * 10 +
                           [C.c_int32, _P, _P, C.c_int64, _P]),
    "gcbf_params_t_count_l": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32]),
    "gcbf_prepare_params_l": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _P, _P, _P]),
    "gcbf_rollout_workspace_floats_l": (C.c_int64, [C.POINTER(EnvDesc), C.c_int32]),
    "gcbf_rollout_step_l": (C.c_int32, [C.POINTER(EnvDesc), C.c_int32, _P, _P, C.c_int32] + [_P] * 21 + [C.c_int64, _P]),
    "gcbf_infer_count": (C.c_int32, [C.c_int32, C.c_int32]),
    "gcbf_prepare_infer": (C.c_int32, [C.c_int32, C.c_int32, _P, _P, _P]),
    "gcbf_gnn_infer": (C.c_int32, [C.POINTER(EnvDesc), C.c_int32, C.c_int32, _P, _P, C.c_int32] + [_P] * 8 +
                       [C.c_int32, _P, _P, C.c_int64, _P]),
    "gcbf_rollout_step_select": (C.c_int32, [C.POINTER(EnvDesc), _P, _P, C.c_int32] + [_P] * 21 + [C.c_int64, C.c_int32, _P]),
    "gcbf_rollout_persistent_workspace_floats": (C.c_int64, [C.POINTER(EnvDesc)]),
    "gcbf_rollout_persistent_supported": (C.c_int32, [C.POINTER(EnvDesc)]),
    "gcbf_rollout_persistent_max_clusters": (C.c_int32, [C.c_int32]),
    "gcbf_rollout_persistent": (C.c_int32, [C.POINTER(EnvDesc), C.c_int32] + [_P] * 12 + [C.c_int64, _P, _P]),
    "gcbf_rollout_persistent_multi": (C.c_int32, [C.POINTER(EnvDesc), C.c_int32, C.c_int32] + [_P] * 13 +
                                      [C.c_int64, _P, _P]),
    "gcbf_rollout_persistent_multi_strides": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(C.c_int64),
                                                          C.POINTER(C.c_int64)]),
    "gcbf_env_step": (C.c_int32, [C.POINTER(EnvDesc)] + [_P] * 11 + [C.c_int32, _P]),
    "gcbf_act": (C.c_int32, [C.POINTER(EnvDesc)] + [_P] * 5),
    "gcbf_masks": (C.c_int32, [C.POINTER(EnvDesc)] + [_P] * 9),
    "gcbf_safe_horizon": (C.c_int32, [_P, _P, C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P]),
    "gcbf_gemm_nn": (C.c_int32, [C.c_int32, C.c_int32] + [_P] * 7 + [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P]),
    "gcbf_gemm_tc": (C.c_int32, [C.c_int32, C.c_int32] + [_P] * 8 + [C.c_int32] * 5 + [_P]),
    "gcbf_split_tf32": (C.c_int32, [_P, _P, _P, C.c_int32, _P]),
    "gcbf_gemm_tn": (C.c_int32, [_P, C.c_int32] + [_P] * 5 + [C.c_int32] * 5 + [_P]),
    "gcbf_gemm_tn_tc": (C.c_int32, [_P, C.c_int32] + [_P] * 5 + [C.c_int32] * 5 + [_P] * 3),
    "gcbf_colsum": (C.c_int32, [_P] * 5 + [C.c_int32] * 4 + [_P]),
    "gcbf_train_workspace_floats": (C.c_int64, [C.POINTER(EnvDesc)]),
    "gcbf_mask_counts": (C.c_int32, [_P, _P, C.c_int32, _P, _P]),
    "gcbf_train_step": (C.c_int32, [C.POINTER(EnvDesc), C.POINTER(C.c_float)] + [_P] * 18 + [C.c_int64, _P]),
    "gcbf_grad_sqnorm": (C.c_int32, [_P, C.c_int32, _P, _P]),
    "gcbf_clip_adamw": (C.c_int32, [_P, _P, _P, _P, C.c_int32, _P, _P, C.c_float, C.c_float, C.c_float, C.c_float,
                                    C.c_float, C.c_float, _P]),
    "gcbf_polyak": (C.c_int32, [_P, _P, C.c_int32, C.c_float, _P]),
    "gcbf_reset_positions": (C.c_int32, [C.POINTER(EnvDesc), _P, _P, C.c_float, C.c_float, C.c_float, _P, _P, _P]),
    "gcbf_reset_positions_ex": (C.c_int32, [C.POINTER(EnvDesc), _P, _P, C.c_float, C.c_float, C.c_float, C.c_int32, _P, _P,
                                            _P]),
    "gcbf_qp_workspace_floats": (C.c_int64, [C.POINTER(EnvDesc)]),
    "gcbf_qp_workspace_layout": (C.c_int32, [C.POINTER(EnvDesc), C.POINTER(C.c_int64)]),
    "gcbf_qp_labels": (C.c_int32, [C.POINTER(EnvDesc), C.c_float, C.c_int32, C.c_int32, C.c_float] + [_P] * 13 +
                       [C.c_int64, _P]),
    "gcbf_qp_filter": (C.c_int32, [C.POINTER(EnvDesc), C.c_float, C.c_int32, C.c_int32, C.c_float] + [_P] * 14 +
                       [C.c_int64, _P]),
    "gcbf_refine_prepare": (C.c_int32, [C.c_int32, C.c_int32, _P, _P, _P]),
    "gcbf_refine_workspace_floats": (C.c_int64, [C.POINTER(EnvDesc)]),
    "gcbf_refine_actions": (C.c_int32, [C.POINTER(EnvDesc), C.c_float, C.c_float, C.c_int32, C.c_int32] + [_P] * 15 +
                            [C.c_int64, _P]),
    "gcbf_cbf_condition_prepare": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int64, _P]),
    "gcbf_cbf_condition_workspace_floats": (C.c_int64, [C.POINTER(EnvDesc)]),
    "gcbf_cbf_condition": (C.c_int32, [C.POINTER(EnvDesc), C.c_float, C.c_int32] + [_P] * 17 + [C.c_int64, _P]),
    "gcbf_cbf_pairwise": (C.c_int32, [C.POINTER(EnvDesc)] + [_P] * 9),
    "gcbf_cbfqp_workspace_floats": (C.c_int64, [C.POINTER(EnvDesc)]),
    "gcbf_cbfqp_dec_share": (C.c_int32, [C.POINTER(EnvDesc), C.c_float, C.c_int32, C.c_float] + [_P] * 7 +
                             [C.c_int64, _P]),
    "gcbf_cbfqp_centralized": (C.c_int32, [C.POINTER(EnvDesc), C.c_float, C.c_int32, C.c_float] + [_P] * 7 +
                               [C.c_int64, _P]),
}


def lib_path() -> str:
    return _LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load (building in-tree with nvcc if needed).  Raises RuntimeError on failure."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        if not build_if_missing:
            raise RuntimeError(f"{_LIB_PATH} is missing: run `python -m gcbfplus_b200.build`")
        from . import build as _build
        _build.build()
    try:
        lib = C.CDLL(_LIB_PATH)
    except OSError as e:  # pragma: no cover
        raise RuntimeError(f"cannot load {_LIB_PATH}: {e}") from e
    for name, (res, args) in _SIGNATURES.items():
        try:
            fn = getattr(lib, name)
        except AttributeError:
            continue  # symbol list is checked by tests/test_abi.py against the header
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(rc: int, what: str = "") -> None:
    if rc != 0:
        msg = load().gcbf_last_error_string().decode(errors="replace")
        raise RuntimeError(f"libgcbf_b200 {what} failed (status {rc}): {msg}")


def ptr(t) -> int:
    """Device pointer of a torch tensor (None -> NULL).  Tensors must be contiguous."""
    if t is None:
        return None
    assert t.is_contiguous(), "non-contiguous tensor passed to libgcbf_b200"
    return t.data_ptr()


#: Bit 30 of an iteration word (`iters` of the device QPs and of the refinement): the bits below it count iterations.
#: What the bit flags depends on the entry point (include/gcbf_b200.h): the dense-graph path for gcbf_qp_labels and
#: gcbf_qp_filter, a solve that hit its cap for gcbf_cbfqp_* and gcbf_refine_actions.
ITER_FLAG = 1 << 30


def split_iters(iters):
    """(iteration counts, flag bits set) of a tensor or array of iteration words."""
    return iters & (ITER_FLAG - 1), (iters & ITER_FLAG) != 0


def f32(v: float) -> float:
    """Round a python double to fp32 (where JAX's weak typing rounds a python scalar)."""
    return float(np.float32(v))


def sqrt_threshold(r: float) -> float:
    """Smallest fp32 a such that the correctly rounded fp32 sqrt(a) >= fp32(r), i.e.
    (sqrtf(x) < r) == (x < a) for every fp32 x >= 0: lets the kernels drop the sqrt bit-exactly."""
    r32 = np.float32(r)
    a = np.float32(r32 * r32)
    while np.sqrt(a) >= r32:
        a = np.nextafter(a, np.float32(0), dtype=np.float32)
    while np.sqrt(a) < r32:
        a = np.nextafter(a, np.float32(np.inf), dtype=np.float32)
    return float(a)


def param_offsets(edge_dim: int, out_dim: int, n_layers: int = 1):
    """W, b offsets of the Dense layers in forward order (gcbf_param_offsets_l): 2 * (9 n_layers + 3) entries."""
    arr = (C.c_int32 * (2 * (9 * n_layers + 3)))()
    check(load().gcbf_param_offsets_l(edge_dim, out_dim, n_layers, arr), "gcbf_param_offsets_l")
    return list(arr)


#: use the wgmma tensor-core GEMMs (3xTF32 split, fp32-class accuracy) instead of the SIMT fp32 GEMMs.
#: GCBF_TENSOR_CORES=0 selects the strict-fp32 SIMT path.
USE_TC = os.environ.get("GCBF_TENSOR_CORES", "1") != "0"


def param_count(edge_dim: int, out_dim: int, n_layers: int = 1) -> int:
    n = load().gcbf_param_count_l(edge_dim, out_dim, n_layers)
    if n <= 0:
        raise RuntimeError(f"gcbf_param_count_l: bad dims (edge_dim {edge_dim}, out_dim {out_dim}, n_layers {n_layers})")
    return int(n)
