"""The CBF-QP baseline controllers the GCBF+ paper compares against: DecShareCBF (gcbfplus/algo/dec_share_cbf.py) and
CentralizedCBF (gcbfplus/algo/centralized_cbf.py), with the pairwise CBFs of gcbfplus/algo/utils.py:44-439 (k = 3).

They have no parameters: act(graph) solves a CBF-QP per agent (DecShareCBF) or per graph (CentralizedCBF) on the
device (csrc/cbfqp.cu).  The reference solves with JaxProxQP capped at 100 iterations; here the QP's unique minimiser
is computed exactly on its dual, with an iteration cap of its own that is reported, never silent (`last_iters`,
`iter_stats`).  Graphs are batched: [G, N, ...] where the reference handles one graph at a time."""
from __future__ import annotations

import ctypes as C
from typing import Optional, Tuple

import numpy as np
import torch

from .. import _lib
from ..env.base import MultiAgentEnv
from ..utils.graph import SwarmGraph
from .base import MultiAgentController

K_NEAREST = 3
#: default iteration cap and stopping threshold (projected dual-gradient residual) of the device QP solves
QP_MAX_ITER = 10000
QP_TOL = 1e-8


def iter_stats(iters: torch.Tensor, cap: Optional[int] = None) -> dict:
    """Median / max iterations and the number of capped solves of an iteration record (`iters` of gcbf_cbfqp_* or
    gcbf_refine_actions, whose bit 30 marks a capped solve).  For gcbf_qp_labels / gcbf_qp_filter, whose bit 30 marks
    the dense-graph path instead, pass their iteration cap: a solve then counts as capped when it ran `cap` iterations."""
    n, flag = _lib.split_iters(iters.reshape(-1).to(torch.int64).cpu().numpy())
    capped = flag if cap is None else n >= cap
    return {"solves": int(n.size), "iters_median": float(np.median(n)) if n.size else 0.0,
            "iters_max": int(n.max()) if n.size else 0, "capped": int(capped.sum())}


class _PairwiseCBFQP(MultiAgentController):
    NAME = ""

    def __init__(self, env: MultiAgentEnv, node_dim: int, edge_dim: int, state_dim: int, action_dim: int,
                 n_agents: int, alpha: float = 1.0, max_iter: int = QP_MAX_ITER, tol: float = QP_TOL, **kwargs):
        super().__init__(env=env, node_dim=node_dim, edge_dim=edge_dim, action_dim=action_dim, n_agents=n_agents)
        self.alpha = float(alpha)
        self.k = K_NEAREST
        self.max_iter = int(max_iter)
        self.tol = float(tol)
        #: iteration record of the last get_qp_action (one entry per solve, bit 30 = capped: _lib.split_iters)
        self.last_iters: Optional[torch.Tensor] = None

    @property
    def env(self) -> MultiAgentEnv:
        return self._env

    @property
    def config(self) -> dict:
        return {"alpha": self.alpha}

    @property
    def actor_params(self):
        raise NotImplementedError(f"{self.NAME} has no parameters")

    def step(self, graph, key=None, params=None):
        raise NotImplementedError(f"{self.NAME} is not a stochastic policy")

    def update(self, rollout, step: int) -> dict:
        raise NotImplementedError(f"{self.NAME} is not trainable")

    def save(self, save_dir: str, step: int):
        raise NotImplementedError(f"{self.NAME} has no parameters to save")

    def load(self, load_dir: str, step: int):
        raise NotImplementedError(f"{self.NAME} has no parameters to load")

    # ------------------------------------------------------------------ device calls
    def _desc(self, graph: SwarmGraph):
        env = self._env
        return env.desc(graph.n_graphs, 0, edge_cap=1)

    def pairwise(self, graph: SwarmGraph, with_other: bool = True) -> dict:
        """Pairwise CBFs of every agent and the Lie terms of their Jacobian (gcbf_cbf_pairwise):
        idx, isobs, h, lf_h [G, N, 3]; lg_self, lg_other [G, N, 3, nu]."""
        env = self._env
        G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
        dev = graph.agent.device
        f32 = dict(dtype=torch.float32, device=dev)
        out = {"idx": torch.empty(G, N, 3, dtype=torch.int32, device=dev),
               "isobs": torch.empty(G, N, 3, dtype=torch.uint8, device=dev),
               "h": torch.empty(G, N, 3, **f32), "lf_h": torch.empty(G, N, 3, **f32),
               "lg_self": torch.empty(G, N, 3, nu, **f32),
               "lg_other": torch.empty(G, N, 3, nu, **f32) if with_other else None}
        d = self._desc(graph)
        rc = env.lib.gcbf_cbf_pairwise(C.byref(d), _lib.ptr(graph.agent.contiguous()), _lib.ptr(graph.hits.contiguous()),
                                       *[_lib.ptr(out[k]) for k in ("idx", "isobs", "h", "lf_h", "lg_self", "lg_other")],
                                       env._stream())
        _lib.check(rc, "gcbf_cbf_pairwise")
        out["isobs"] = out["isobs"].bool()
        return out

    def _solve(self, graph: SwarmGraph) -> Tuple[torch.Tensor, torch.Tensor]:
        env = self._env
        G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
        dev = graph.agent.device
        d = self._desc(graph)
        n_ws = int(env.lib.gcbf_cbfqp_workspace_floats(C.byref(d)))
        ws = torch.empty(max(n_ws, 1), dtype=torch.float32, device=dev)
        u = torch.empty(G, N, nu, dtype=torch.float32, device=dev)
        r = torch.empty(G, N, 3, dtype=torch.float32, device=dev)
        iters = torch.empty(self._n_solves(G, N), dtype=torch.int32, device=dev)
        fn = getattr(env.lib, self._ENTRY)
        rc = fn(C.byref(d), self.alpha, self.max_iter, self.tol, _lib.ptr(graph.agent.contiguous()),
                _lib.ptr(graph.goal.contiguous()), _lib.ptr(graph.hits.contiguous()), _lib.ptr(u), _lib.ptr(r),
                _lib.ptr(iters), _lib.ptr(ws), ws.numel(), env._stream())
        _lib.check(rc, self._ENTRY)
        self.last_iters = iters
        return u, r

    # ------------------------------------------------------------------ reference surface
    def get_qp_action(self, graph: SwarmGraph, relax_penalty: float = 1e3) -> Tuple[torch.Tensor, torch.Tensor]:
        """(u [G, N, nu], r [G, N, 3]): the QP's minimiser and relaxations."""
        if relax_penalty != 1e3:
            raise ValueError("the device QP uses the reference's relax_penalty = 1e3")
        return self._solve(graph)

    def act(self, graph: SwarmGraph, params=None) -> torch.Tensor:
        return self.get_qp_action(graph)[0]

    def iter_stats(self) -> dict:
        """Iteration statistics of the last get_qp_action."""
        if self.last_iters is None:
            raise RuntimeError("no QP has been solved yet")
        return iter_stats(self.last_iters)


class DecShareCBF(_PairwiseCBFQP):
    """gcbfplus/algo/dec_share_cbf.py: one QP per agent over its own action and 3 relaxations, each CBF row scaled by
    its responsibility (1 for an obstacle, 0.5 for an agent).  Turns the DubinsCar stop mask off (:34-35)."""
    NAME = "dec_share_cbf"
    _ENTRY = "gcbf_cbfqp_dec_share"

    def __init__(self, env: MultiAgentEnv, *args, **kwargs):
        super().__init__(env, *args, **kwargs)
        if hasattr(env, "enable_stop"):
            env.enable_stop = False

    @staticmethod
    def _n_solves(G: int, N: int) -> int:
        return G * N

    def get_cbf(self, graph: SwarmGraph) -> Tuple[torch.Tensor, torch.Tensor]:
        """(h, isobs) [G, N, 3]."""
        p = self.pairwise(graph, with_other=False)
        return p["h"], p["isobs"]


class CentralizedCBF(_PairwiseCBFQP):
    """gcbfplus/algo/centralized_cbf.py: one QP per graph over all actions and 3N relaxations."""
    NAME = "centralized_cbf"
    _ENTRY = "gcbf_cbfqp_centralized"
    MAX_AGENTS = 1024   # GCBF_CBFQP_CENTRAL_MAX_AGENTS (include/gcbf_b200.h): the per-graph QP lives in shared memory

    def __init__(self, env: MultiAgentEnv, *args, **kwargs):
        super().__init__(env, *args, **kwargs)
        limit = 999 if env.action_dim == 3 else self.MAX_AGENTS
        if env.num_agents > limit:
            raise ValueError(f"centralized_cbf supports at most {limit} agents per graph in {type(env).__name__} "
                             f"(got {env.num_agents})")

    @staticmethod
    def _n_solves(G: int, N: int) -> int:
        return G

    def get_cbf(self, graph: SwarmGraph) -> torch.Tensor:
        """h [G, N, 3]."""
        return self.pairwise(graph, with_other=False)["h"]


BASELINES = {DecShareCBF.NAME: DecShareCBF, CentralizedCBF.NAME: CentralizedCBF}
