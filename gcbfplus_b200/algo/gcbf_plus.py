"""GCBFPlus -- host-side mirror of gcbfplus/algo/gcbf_plus.py (and the pieces it inherits from
gcbfplus/algo/gcbf.py: get_cbf, save, load, actor_params).  All arithmetic is in
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
        from .train import qp_labels
        u, aux, _ = qp_labels(self, graph, params=cbf_params or self.cbf_params, with_aux=True)
        return u, aux[..., 1]

    def get_b_u_qp(self, b_graph: SwarmGraph, params: Optional[NetParams] = None) -> torch.Tensor:
        """gcbf_plus.py:193-196."""
        from .train import qp_labels
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
