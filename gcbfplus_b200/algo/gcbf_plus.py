"""GCBFPlus -- host-side mirror of gcbfplus/algo/gcbf_plus.py (and the pieces it inherits from
gcbfplus/algo/gcbf.py: get_cbf, online_policy_refinement, save, load, actor_params).  All arithmetic is in
libgcbf_b200.so; this file is orchestration: parameter buffers, replay, minibatching.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional, Tuple

import numpy as np
import torch

from .. import _lib
from ..env.base import MultiAgentEnv
from ..utils.graph import SwarmGraph
from .base import MultiAgentController
from .nets import GnnRunner
from .params import NetParams
from .refine import (REFINE_LR, REFINE_MAX_ITER, launch_refine, planes_buffer, prepare_planes, refine_workspace,
                     require_one_layer_refine)
from .train import QP_MAX_ITER, QP_TOL, qp_labels


class GCBFPlus(MultiAgentController):

    def __init__(self, env: MultiAgentEnv, node_dim: int, edge_dim: int, state_dim: int, action_dim: int,
                 n_agents: int, gnn_layers: int = 1, batch_size: int = 256, buffer_size: int = 512,
                 horizon: int = 32, lr_actor: float = 3e-5, lr_cbf: float = 3e-5, alpha: float = 1.0,
                 eps: float = 0.02, inner_epoch: int = 8, loss_action_coef: float = 0.001,
                 loss_unsafe_coef: float = 1.0, loss_safe_coef: float = 1.0, loss_h_dot_coef: float = 0.2,
                 max_grad_norm: float = 2.0, seed: int = 0, **kwargs):
        """Same kwargs as gcbf_plus.py:36-60."""
        super().__init__(env=env, node_dim=node_dim, edge_dim=edge_dim, action_dim=action_dim, n_agents=n_agents)
        if gnn_layers < 1:
            raise ValueError(f"gnn_layers must be >= 1, got {gnn_layers}")
        self.batch_size = batch_size
        self.buffer_size = buffer_size
        self.lr_actor = lr_actor
        self.lr_cbf = lr_cbf
        self.alpha = alpha
        self.eps = eps
        self.inner_epoch = inner_epoch
        self.loss_action_coef = loss_action_coef
        self.loss_unsafe_coef = loss_unsafe_coef
        self.loss_safe_coef = loss_safe_coef
        self.loss_h_dot_coef = loss_h_dot_coef
        self.gnn_layers = gnn_layers
        self.max_grad_norm = max_grad_norm
        self.seed = seed
        self.horizon = horizon
        self.state_dim = state_dim
        dev = env.device
        # gcbf_plus.py:98-133: cbf, target cbf (copy), actor; xavier-uniform init (NumPy PCG64 stream)
        self.cbf_params = NetParams(edge_dim, 1, "cbf", device=dev, n_layers=gnn_layers).init_xavier(seed * 2 + 1)
        self.cbf_tgt_params = self.cbf_params.clone()
        self.actor_net_params = NetParams(edge_dim, action_dim, "actor", device=dev,
                                          n_layers=gnn_layers).init_xavier(seed * 2 + 2)
        self.runner = GnnRunner(env)
        self.rng = np.random.default_rng(seed=seed + 1)       # gcbf_plus.py:139
        self._trainer_state = None                            # lazily built by update() (algo/train.py)
        # online_policy_refinement: the CBF's prepared planes (rebuilt on every call) and the workspace of the last
        # batch shape (n_graphs, edge_cap)
        self._refine_planes = planes_buffer(self.cbf_params)
        self._refine_ws: Optional[torch.Tensor] = None
        self._refine_ws_key = None

    # ------------------------------------------------------------------ reference surface
    @property
    def config(self) -> dict:
        """gcbf_plus.py:141-158."""
        return {
            "batch_size": self.batch_size, "lr_actor": self.lr_actor, "lr_cbf": self.lr_cbf, "alpha": self.alpha,
            "eps": self.eps, "inner_epoch": self.inner_epoch, "loss_action_coef": self.loss_action_coef,
            "loss_unsafe_coef": self.loss_unsafe_coef, "loss_safe_coef": self.loss_safe_coef,
            "loss_h_dot_coef": self.loss_h_dot_coef, "gnn_layers": self.gnn_layers, "seed": self.seed,
            "max_grad_norm": self.max_grad_norm, "horizon": self.horizon,
        }

    @property
    def actor_params(self) -> NetParams:
        return self.actor_net_params

    def get_action(self, graph: SwarmGraph, params: Optional[NetParams] = None) -> torch.Tensor:
        """DeterministicPolicy.get_action (policy.py:127-128): pi(g) in (-1, 1), [G, N, nu]."""
        return self.runner.forward(params or self.actor_net_params, graph)

    def act(self, graph: SwarmGraph, params: Optional[NetParams] = None) -> torch.Tensor:
        """gcbf_plus.py:176-180: 2 * pi(g) + u_ref(g)."""
        pi = self.get_action(graph, params)
        env = self._env
        d = env.desc(graph.n_graphs, 0, edge_cap=graph.edge_recv.numel())
        out = torch.empty_like(pi)
        _lib.check(env.lib.gcbf_act(C.byref(d), _lib.ptr(graph.agent), _lib.ptr(graph.goal), _lib.ptr(pi),
                                    _lib.ptr(out), env._stream()), "gcbf_act")
        return out

    def step(self, graph: SwarmGraph, key=None, params: Optional[NetParams] = None) -> Tuple[torch.Tensor, torch.Tensor]:
        """gcbf_plus.py:182-186 (deterministic policy: log_pi = 0, policy.py:130-133)."""
        action = self.act(graph, params)
        return action, torch.zeros_like(action)

    def online_policy_refinement(self, graph: SwarmGraph, params: Optional[NetParams] = None, *,
                                 lr: float = REFINE_LR, max_iter: int = REFINE_MAX_ITER, return_info: bool = False):
        """gcbf.py:161-201 for every graph of the batch: the action 2 pi + u_ref (or u_ref where u_ref alone keeps the
        CBF condition) refined by gradient steps on mean_agents relu(-h_dot - alpha h) of the next graph until that
        value is 0 or max_iter steps were taken; each graph stops on its own.  params: the actor's parameters.
        Returns actions [G, N, nu]; with return_info also (value [G], iters [G]): the last loop value and the steps
        taken (bit 30 set where a graph stopped at max_iter with value > 0)."""
        env = self._env
        actor = params or self.actor_net_params
        require_one_layer_refine(actor, "actor")
        require_one_layer_refine(self.cbf_params, "CBF")
        pi = self.get_action(graph, actor)
        G = graph.n_graphs
        d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
        stream = env._stream()
        if self._refine_ws_key != (G, d.edge_cap):
            self._refine_ws = None
            self._refine_ws = refine_workspace(env, d)
            self._refine_ws_key = (G, d.edge_cap)
        # the planes of the parameters as they are now (one launch; the optimizer writes them through raw pointers)
        use_tc = 1 if _lib.USE_TC else 0
        prepared = prepare_planes(self.cbf_params, self._refine_planes, use_tc, stream)
        action = torch.empty_like(pi)
        value = torch.empty(G, dtype=torch.float32, device=pi.device)
        iters = torch.empty(G, dtype=torch.int32, device=pi.device)
        launch_refine(env, d, self.alpha, lr, max_iter, use_tc, self.cbf_params, prepared, pi, graph.agent, graph.goal,
                      graph.hits, graph.row_start, graph.row_deg, graph.edge_recv, graph.edge_src, graph.counters,
                      action, value, iters, self._refine_ws, stream)
        if return_info:
            return action, value, iters
        return action

    def get_cbf(self, graph: SwarmGraph, params: Optional[NetParams] = None) -> torch.Tensor:
        """gcbf.py:209-212 -> [G, N, 1]."""
        return self.runner.forward(params or self.cbf_params, graph)

    def get_qp_action(self, graph: SwarmGraph, relax_penalty: float = 1e3, cbf_params: Optional[NetParams] = None,
                      qp_settings=None) -> Tuple[torch.Tensor, torch.Tensor]:
        """gcbf_plus.py:299-352 for every graph of the batch: (u_opt [G, N, nu], relaxation r [G, N]).
        relax_penalty is fixed at the reference's 1e3 in the kernel; qp_settings is accepted and ignored
        (the device solver has its own iteration cap / tolerance, algo/train.py)."""
        if relax_penalty != 1e3:
            raise NotImplementedError("relax_penalty is compiled in (1e3, gcbf_plus.py:302)")
        u, aux, _ = qp_labels(self, graph, params=cbf_params or self.cbf_params, with_aux=True)
        return u, aux[..., 1]

    def safety_filter(self, graph: SwarmGraph, u_nom: Optional[torch.Tensor] = None, *,
                      cbf_params: Optional[NetParams] = None, max_iter: int = QP_MAX_ITER, tol: float = QP_TOL,
                      return_info: bool = False):
        """The learned CBF as a QP safety filter, for every graph of the batch: the action closest to the nominal
        u_nom [G, N, nu] (default u_ref: then this is get_qp_action) such that the CBF condition
        Lf_h + Lg_h u + 0.1 alpha h >= 0 holds, relaxed by r >= 0 at cost 1000 r + 5 r^2 where no action in the u_lim
        box satisfies it.  cbf_params defaults to the CBF itself (not the target network); alpha is self.alpha.
        Returns u [G, N, nu]; with return_info also (r [G, N], iters [G]): a graph whose count reaches max_iter stopped
        at the cap and its action is the capped iterate."""
        u, aux, iters = qp_labels(self, graph, params=cbf_params or self.cbf_params, with_aux=True,
                                  max_iter=max_iter, tol=tol, u_nom=u_nom)
        if return_info:
            return u, aux[..., 1], iters
        return u

    def get_b_u_qp(self, b_graph: SwarmGraph, params: Optional[NetParams] = None) -> torch.Tensor:
        """gcbf_plus.py:193-196."""
        return qp_labels(self, b_graph, params=params or self.cbf_tgt_params)

    def update(self, rollout, step: int) -> dict:
        from .train import update as _update
        return _update(self, rollout, step)

    def save(self, save_dir: str, step: int):
        """gcbf.py:344-349: <dir>/<step>/{actor,cbf}.pkl = pickled {'params': nested dict}."""
        model_dir = os.path.join(save_dir, str(step))
        os.makedirs(model_dir, exist_ok=True)
        self.actor_net_params.save(os.path.join(model_dir, "actor.pkl"))
        self.cbf_params.save(os.path.join(model_dir, "cbf.pkl"))

    def load(self, load_dir: str, step: int):
        """gcbf.py:351-357 (also reads the reference's own jax.Array pickles)."""
        path = os.path.join(load_dir, str(step))
        self.actor_net_params.load(os.path.join(path, "actor.pkl"))
        self.cbf_params.load(os.path.join(path, "cbf.pkl"))

    def load_npz(self, npz_path: str):
        """Load a tests/golden/params_<Env>.npz fixture (flattened reference pickles)."""
        from .params import unflatten_tree
        z = np.load(npz_path)
        self.actor_net_params.from_tree(unflatten_tree({k[6:]: z[k] for k in z.files if k.startswith("actor:")}))
        self.cbf_params.from_tree(unflatten_tree({k[4:]: z[k] for k in z.files if k.startswith("cbf:")}))
        self.cbf_tgt_params.flat.copy_(self.cbf_params.flat)
