"""Online policy refinement of GCBF+ (gcbfplus/algo/gcbf.py:161-201) on the device: gcbf_refine_actions.

The policy's action is corrected by gradient steps on the CBF condition of the next graph until it holds, per graph
and with the reference's constants (lr = 0.1, at most 30 steps).  Used by GCBFPlus.online_policy_refinement and by the
rollout engine's `actor_refine` policy (test.py --online-refine)."""
from __future__ import annotations

import ctypes as C

import torch

from .. import _lib
from .params import NetParams

REFINE_LR = 0.1
REFINE_MAX_ITER = 30


def require_one_layer_refine(params: NetParams, what: str) -> None:
    """The refinement's backward is the one-layer data-only CBF backward (DESIGN 6)."""
    if params.n_layers != 1:
        raise NotImplementedError(f"online policy refinement implements gnn_layers = 1; the {what} has "
                                  f"{params.n_layers} GNN layers")


def planes_buffer(params: NetParams) -> torch.Tensor:
    """A buffer for the CBF's prepared planes (gcbf_params_t_count_l(edge_dim, 1, 1) floats: enough for either GEMM
    path)."""
    n = _lib.load().gcbf_params_t_count_l(params.edge_dim, 1, 1)
    return torch.empty(int(n), dtype=torch.float32, device=params.flat.device)


def prepare_planes(params: NetParams, planes: torch.Tensor, use_tc: int, stream: int) -> torch.Tensor:
    """Enqueue gcbf_refine_prepare: the planes of the CURRENT `params.flat` (tf32 planes on the tensor-core path,
    transposed weights on the strict-fp32 path) into `planes`.  Always rebuilt: the project's optimizer and polyak
    kernels write the parameters through raw pointers, so no host-side cache key can tell that they changed."""
    require_one_layer_refine(params, "CBF")
    _lib.check(_lib.load().gcbf_refine_prepare(params.edge_dim, int(use_tc), _lib.ptr(params.flat),
                                               _lib.ptr(planes), stream), "gcbf_refine_prepare")
    return planes


def refine_workspace(env, desc: _lib.EnvDesc) -> torch.Tensor:
    n = env.lib.gcbf_refine_workspace_floats(C.byref(desc))
    if n <= 0:
        raise RuntimeError("gcbf_refine_workspace_floats: bad descriptor")
    return torch.empty(int(n), dtype=torch.float32, device=env.device)


def launch_refine(env, desc: _lib.EnvDesc, alpha: float, lr: float, max_iter: int, use_tc: int, cbf: NetParams,
                  prepared: torch.Tensor, pi, agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters,
                  action, value, iters, ws: torch.Tensor, stream: int) -> None:
    """Enqueue gcbf_refine_actions (no host sync); `prepared` must come from prepare_planes with the same use_tc."""
    if int(max_iter) < 1:
        raise ValueError(f"max_iter must be >= 1, got {max_iter}")
    rc = env.lib.gcbf_refine_actions(C.byref(desc), float(alpha), float(lr), int(max_iter), int(use_tc),
                                     _lib.ptr(cbf.flat), _lib.ptr(prepared), _lib.ptr(pi), _lib.ptr(agent),
                                     _lib.ptr(goal), _lib.ptr(hits), _lib.ptr(row_start), _lib.ptr(row_deg),
                                     _lib.ptr(edge_recv), _lib.ptr(edge_src), _lib.ptr(counters), _lib.ptr(action),
                                     _lib.ptr(value), _lib.ptr(iters), _lib.ptr(ws), ws.numel(), stream)
    _lib.check(rc, "gcbf_refine_actions")
