"""Forward evaluation of the two GNN networks through libgcbf_b200 (gcbf_gnn_forward_l)."""
from __future__ import annotations

import ctypes as C
from typing import Dict, Optional, Tuple

import torch

from .. import _lib
from ..utils.graph import SwarmGraph
from .params import NetParams


class GnnRunner:
    """Owns the activation workspace for one (env, batch shape) and runs a network forward.
    Replaces CBF.get_cbf / DeterministicPolicy.get_action (algo/module/cbf.py:52-53,
    algo/module/policy.py:127-128)."""

    def __init__(self, env):
        self.env = env
        self._ws: Dict[Tuple[int, int], torch.Tensor] = {}

    def workspace(self, desc: _lib.EnvDesc, out_dim: int, device, n_layers: int = 1) -> torch.Tensor:
        key = (desc.n_graphs, desc.edge_cap) if n_layers == 1 else (desc.n_graphs, desc.edge_cap, n_layers)
        ws = self._ws.get(key)
        if ws is None or ws.device != device:
            n = self.env.lib.gcbf_gnn_workspace_floats_l(C.byref(desc), out_dim, n_layers)
            if n <= 0:
                raise RuntimeError("gcbf_gnn_workspace_floats_l failed")
            ws = torch.empty(int(n), dtype=torch.float32, device=device)
            self._ws[key] = ws
        return ws

    def forward(self, params: NetParams, graph: SwarmGraph, out: Optional[torch.Tensor] = None,
                workspace: Optional[torch.Tensor] = None) -> torch.Tensor:
        env = self.env
        G, N = graph.n_graphs, env.num_agents
        d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
        dev = graph.agent.device
        if out is None:
            out = torch.empty(G, N, params.out_dim, dtype=torch.float32, device=dev)
        ws = workspace if workspace is not None else self.workspace(d, params.out_dim, dev, params.n_layers)
        kind = _lib.NET_CBF if params.kind == "cbf" else _lib.NET_ACTOR
        rc = env.lib.gcbf_gnn_forward_l(C.byref(d), kind, params.out_dim, params.n_layers, _lib.ptr(params.flat),
                                        _lib.ptr(params.prepared(env._stream())), _lib.ptr(graph.agent),
                                        _lib.ptr(graph.goal), _lib.ptr(graph.hits), _lib.ptr(graph.row_start),
                                        _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_recv), _lib.ptr(graph.edge_src),
                                        _lib.ptr(graph.counters), 1 if graph.clip_all else 0, _lib.ptr(out),
                                        _lib.ptr(ws), ws.numel(), env._stream())
        _lib.check(rc, "gcbf_gnn_forward_l")
        return out
