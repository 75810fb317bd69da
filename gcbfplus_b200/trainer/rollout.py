"""Batched closed-loop rollout -- replaces jit(vmap(rollout)) of gcbfplus/trainer/utils.py:25-55
and trainer/trainer.py:81-87.

Two device paths with the same arithmetic (bit-identical results, tests/test_gpu_rollout.py):
* persistent (default where supported: 2-D environments, n <= 512): ONE kernel launch for the whole T-step rollout, one
  thread-block cluster per environment looping over the steps (csrc/rollout_persist.cu);
* 5-launch env-step (gcbf_rollout_step_l), the whole T-step loop captured in one CUDA graph: LinearDrone, n > 512,
  GCBF_PERSISTENT=0, the u_ref policy, and actors with more than one GNN layer (the engine takes the depth from the
  network set_params() receives).
No host sync inside the loop on either path.
The CBF-QP baselines (algo/cbf_qp.py) run on the CUDA-graph path: per step the pairwise CBFs + QP solve (2 launches),
env.step with the QP action as input, and the graph build of the next state.
The `actor_refine` policy (GCBF+ with online policy refinement, algo/refine.py) runs on the same path: per step the
policy forward, the refinement of its action against the CBF (gcbf_refine_actions), env.step with the refined action as
input, and the graph build of the next state.
The `actor_qp` and `u_ref_qp` policies (the learned CBF as a QP safety filter, GCBFPlus.safety_filter) run on the same
path: per step the policy forward and its action 2 pi + u_ref (actor_qp) or u_ref (u_ref_qp) as the nominal, the CBF-QP
nearest to it (gcbf_qp_filter), env.step with the filtered action as input, and the canonical graph build of the next
state.
Several actor networks (n_nets > 1; set_params() takes a list): environment g runs network net_of_env[g], by default
g // (n_envs // n_nets).  Where the persistent kernel applies, ONE gcbf_rollout_persistent_multi launch rolls out every
network, each cluster reading its own network's weights, so every network's environments get the bits a solo persistent
rollout of that network gives them.  Otherwise (LinearDrone, n > 512, deeper actors, persistent=False or not chosen by
default) the engine runs one solo engine per network, one after another, and gathers their records.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from .. import _lib
from ..algo.cbf_qp import BASELINES, iter_stats
from ..algo.params import NetParams
from ..algo.refine import (REFINE_LR, REFINE_MAX_ITER, launch_refine, planes_buffer, prepare_planes,
                           refine_workspace, require_one_layer_refine)
from ..algo.train import QP_MAX_ITER, QP_TOL, require_one_layer
from ..utils.graph import SwarmGraph
from .data import Rollout

#: the CBF-QP safety-filter policies: the nominal action of each, filtered by the learned CBF
QP_FILTER_POLICIES = ("actor_qp", "u_ref_qp")


class _Chain:
    """Scratch of the step-by-step path: topology arrays, policy output and activation workspace of all the
    environments (e0 = 0: the first of them)."""

    def __init__(self, eng: "RolloutEngine"):
        env, dev = eng.env, eng.env.device
        self.e0 = 0
        E, N, nu = eng.E, env.num_agents, env.action_dim
        f32, i32 = torch.float32, torch.int32
        self.desc = env.desc(E, eng.O)
        cap = self.desc.edge_cap
        self.pi = torch.zeros(E, N, nu, dtype=f32, device=dev)
        # edge lists are double-buffered: step t reads half t % 2 while the graph of state t+1 is written into the
        # other half (gcbf_rollout_step_l's fused tail + graph build reads the old lists for the step cost)
        self.row_start = torch.zeros(2, E * N, dtype=i32, device=dev)
        self.row_deg = torch.zeros(2, E * N, dtype=i32, device=dev)
        self.edge_recv = torch.zeros(2, cap, dtype=i32, device=dev)
        self.edge_src = torch.zeros(2, cap, dtype=i32, device=dev)
        self.counters = torch.zeros(eng.T + 1, 4, dtype=i32, device=dev)
        n_ws = env.lib.gcbf_rollout_workspace_floats_l(C.byref(self.desc), 1)
        self.ws = torch.empty(int(n_ws), dtype=f32, device=dev)
        if eng.controller is not None:
            # CBF-QP baseline: pairwise-CBF workspace, relaxations (scratch) and the per-step iteration record
            n_qp = env.lib.gcbf_cbfqp_workspace_floats(C.byref(self.desc))
            self.qp_ws = torch.empty(int(n_qp), dtype=f32, device=dev)
            self.qp_r = torch.empty(E, N, 3, dtype=f32, device=dev)
            self.qp_iters = torch.zeros(eng.T, eng.controller._n_solves(E, N), dtype=i32, device=dev)
        if eng.policy == "actor_refine":
            # refinement workspace and the per-step iteration record of every graph
            self.refine_ws = refine_workspace(env, self.desc)
            self.refine_iters = torch.zeros(eng.T, E, dtype=i32, device=dev)
        if eng.policy in QP_FILTER_POLICIES:
            # QP workspace and the per-step record: iterations per graph, nominal actions, (lam, r) per agent
            n_qp = env.lib.gcbf_qp_workspace_floats(C.byref(self.desc))
            if n_qp <= 0:
                raise RuntimeError("gcbf_qp_workspace_floats: bad descriptor")
            self.qp_ws = torch.empty(int(n_qp), dtype=f32, device=dev)
            self.qp_iters = torch.zeros(eng.T, E, dtype=i32, device=dev)
            self.qp_nominal = torch.zeros(eng.T, E, N, nu, dtype=f32, device=dev)
            self.qp_aux = torch.zeros(eng.T, E, N, 2, dtype=f32, device=dev)


def check_net_table(net_of_env, n_nets: int, n_envs: int) -> list:
    """Host check of a network table before any launch: one entry per environment, each in [0, n_nets), and every
    network runs at least one environment.  Returns the table as a list of ints."""
    table = [int(k) for k in net_of_env]
    if len(table) != n_envs:
        raise ValueError(f"net_of_env has {len(table)} entries for {n_envs} environments")
    bad = [k for k in table if not 0 <= k < n_nets]
    if bad:
        raise ValueError(f"net_of_env entry {bad[0]} is out of range for {n_nets} networks")
    idle = sorted(set(range(n_nets)) - set(table))
    if idle:
        raise ValueError(f"network {idle[0]} runs no environment in net_of_env")
    return table


def check_nets(nets, n_nets: int) -> list:
    """The networks of one multi-network rollout: n_nets actors of one edge dim, action dim and depth."""
    nets = [nets] if isinstance(nets, NetParams) else list(nets)
    if len(nets) != n_nets:
        raise ValueError(f"set_params: the engine runs {n_nets} networks, got {len(nets)}")
    for key in ("edge_dim", "out_dim", "n_layers"):
        vals = [getattr(p, key) for p in nets]
        if len(set(vals)) > 1:
            raise ValueError(f"set_params: the networks differ in {key} ({vals})")
    return nets


class RolloutEngine:
    def __init__(self, env, n_envs: int, T: Optional[int] = None, n_obs: Optional[int] = None,
                 use_cuda_graph: bool = True, policy: str = "actor", persistent: Optional[bool] = None,
                 n_nets: int = 1, net_of_env=None):
        """n_nets: number of actor networks (policy 'actor' only).  Environment g runs network net_of_env[g]; the
        default table gives each network n_envs // n_nets consecutive environments (n_envs % n_nets == 0).
        policy: 'actor' (a = 2 pi + u_ref, algo.step), 'actor_refine' (that action refined against the CBF,
        GCBFPlus.online_policy_refinement; set_cbf_params() gives the CBF), 'actor_qp' / 'u_ref_qp' (2 pi + u_ref or
        u_ref filtered by the CBF, GCBFPlus.safety_filter; set_cbf_params() gives the CBF), 'u_ref' (test.py --u-ref), or a CBF-QP
        baseline: a DecShareCBF / CentralizedCBF object, or its name ('dec_share_cbf' / 'centralized_cbf': built with
        alpha = 1)."""
        self.env = env
        self.E = n_envs
        self.T = T or env.max_episode_steps
        self.O = env.params["n_obs"] if n_obs is None else n_obs
        self.controller = None
        if not isinstance(policy, str):
            self.controller, policy = policy, policy.NAME
        elif policy in BASELINES:
            self.controller = BASELINES[policy](env, env.node_dim, env.edge_dim, env.state_dim, env.action_dim,
                                                env.num_agents)
        elif policy not in ("actor", "actor_refine", "u_ref") + QP_FILTER_POLICIES:
            raise ValueError(f"unknown rollout policy {policy!r}")
        if self.controller is None and not getattr(env, "enable_stop", True):
            raise ValueError("the actor / u_ref rollouts apply the DubinsCar stop mask; env.enable_stop is False "
                             "(set by DecShareCBF)")
        self.policy = policy
        self.use_cuda_graph = use_cuda_graph
        self.n_nets = int(n_nets)
        if self.n_nets < 1:
            raise ValueError(f"n_nets must be >= 1, got {n_nets}")
        if self.n_nets > 1 and policy != "actor":
            raise ValueError(f"n_nets > 1 rolls out actor networks (policy 'actor'), not {policy!r}")
        if net_of_env is None:
            if n_envs % self.n_nets:
                raise ValueError(f"n_envs ({n_envs}) must be a multiple of n_nets ({self.n_nets})")
            net_of_env = [g // (n_envs // self.n_nets) for g in range(n_envs)]
        #: the network of every environment (host list) and each network's environments
        self.net_table = check_net_table(net_of_env, self.n_nets, n_envs)
        self.net_envs = [[g for g, k in enumerate(self.net_table) if k == j] for j in range(self.n_nets)]
        # actor_refine / actor_qp / u_ref_qp: a copy of the CBF, its prepared planes (actor_refine) and the settings
        # (set_cbf_params)
        self.cbf_params: Optional[NetParams] = None
        self._refine_planes: Optional[torch.Tensor] = None
        self.refine_alpha, self.refine_lr, self.refine_max_iter = 1.0, REFINE_LR, REFINE_MAX_ITER
        dev = env.device
        E, T, N = self.E, self.T, env.num_agents
        sd, nu, R, pd = env.state_dim, env.action_dim, env.n_hits, env.pos_dim
        f32, i32 = torch.float32, torch.int32
        self.agent = torch.zeros(T + 1, E, N, sd, dtype=f32, device=dev)
        self.hits = torch.zeros(T + 1, E, N, R, pd, dtype=f32, device=dev)
        self.goal = torch.zeros(E, N, sd, dtype=f32, device=dev)
        self.obs_w = 16 if pd == 2 else 4
        self.obstacles = torch.zeros(E, max(self.O, 1), self.obs_w, dtype=f32, device=dev)
        self.actions = torch.zeros(T, E, N, nu, dtype=f32, device=dev)
        self.rewards = torch.zeros(T, E, dtype=f32, device=dev)
        self.costs = torch.zeros(T, E, dtype=f32, device=dev)
        self.chains = [_Chain(self)]   # a one-element list: bench.py reads eng.chains[0]
        self.desc = self.chains[0].desc
        self.params_buf = torch.zeros(_lib.param_count(env.edge_dim, nu), dtype=f32, device=dev)
        # folded inference weights (gcbf_prepare_infer), rebuilt by set_params()
        self.infer_blob = torch.zeros(int(env.lib.gcbf_infer_count(env.edge_dim, nu)), dtype=f32, device=dev)
        self.use_tc = 1 if _lib.USE_TC else 0
        # persistent single-launch rollout (csrc/rollout_persist.cu) where the library supports the configuration
        # the persistent kernel splits the edge capacity evenly over the environments (and, in pair mode, over the pairs
        # of an environment), so it gets a roomier descriptor than the pooled lists of the 5-launch path: 48 rows per
        # agent (or the worst case 1 + (N - 1) + R when that is smaller)
        per_agent = min(1 + (N - 1) + R, max(2 * env.edge_cap_per_agent, 48))
        self._pdesc = env.desc(E, self.O, edge_cap=E * N * per_agent)
        level = int(env.lib.gcbf_rollout_persistent_supported(C.byref(self._pdesc))) \
            if (policy == "actor" and self.use_tc) else 0
        ok = level > 0
        self._persistent_requested = persistent is True   # an explicit request, not the default choice below
        self._persistent_arg = persistent                 # what each per-network engine of a sequential path gets
        if persistent is None:
            # default only where every environment's cluster is resident at once (level 2): otherwise the environments
            # beyond the resident clusters run in a second round
            # DubinsCar is opt-in: its persistent rollout agrees with the 5-launch path only to closed-loop rounding.
            # States and actions are identical while every speed is 0
            # (step 0); from the first step with v != 0 a few policy outputs differ by 1-2 ulp (1.8e-7) -- the
            # (v cos th, v sin th) edge features are evaluated in two translation units -- which the closed loop
            # amplifies to 1.6e-5 after 24 steps.  Env-sharded runs must not mix two numeric paths.
            # Several networks take the persistent kernel at level 1 as well: gcbf_rollout_persistent_multi then runs the
            # clusters beyond the resident ones in later rounds, which is still one launch instead of one per network.
            persistent = (level >= (2 if self.n_nets == 1 else 1) and env.ENV_ID != "DubinsCar"
                          and os.environ.get("GCBF_PERSISTENT", "1") != "0")
        if persistent and not ok:
            raise ValueError("persistent rollout unsupported for this configuration (2-D env, n <= 512, tensor-core path, "
                             "actor policy)")
        self.persistent = bool(persistent)
        self._persistent_one_layer = self.persistent   # the path a one-layer actor takes (restored by _set_depth)
        self.n_layers = 1           # GNN depth of the actor, taken from the network set_params() receives
        #: optional [T + 1, 8] int64 device tensor: in-kernel %globaltimer stamps of the persistent rollout (set before
        #: the first run(); see gcbf_rollout_persistent in include/gcbf_b200.h)
        self.phase_stamps: Optional[torch.Tensor] = None
        self._pws = None
        if self.persistent:
            n = env.lib.gcbf_rollout_persistent_workspace_floats(C.byref(self._pdesc))
            self._pws = torch.empty(int(n), dtype=f32, device=dev)
        # bit 3: rows in ticket order.  The safety filter's sums run over the edge lists in row order, so its policies
        # build canonical graphs: deterministic, and equal to env.get_graph's
        self._build_flags = 1 if policy in QP_FILTER_POLICIES else 1 | 8
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_run = 0
        self._obstacle_obj = None
        if self.n_nets > 1:
            # the network table on the device, the per-network step counters, and -- on the persistent path -- the
            # stacked weights of gcbf_rollout_persistent_multi ([n_nets, stride] each; strides from the library)
            self._net_of_env = torch.tensor(self.net_table, dtype=i32, device=dev)
            self._net_counters = torch.zeros(T + 1, self.n_nets, 4, dtype=i32, device=dev)
            ps, ist = C.c_int64(), C.c_int64()
            _lib.check(env.lib.gcbf_rollout_persistent_multi_strides(env.edge_dim, nu, C.byref(ps), C.byref(ist)),
                       "gcbf_rollout_persistent_multi_strides")
            self._strides = (int(ps.value), int(ist.value))
            self._multi_persistent = self.persistent    # the path one-layer actors take
            self._subs: Optional[list] = None            # the per-network engines of the sequential path
            if self.persistent:
                self.params_buf = torch.zeros(self.n_nets, self._strides[0], dtype=f32, device=dev)
                self.infer_blob = torch.zeros(self.n_nets, self._strides[1], dtype=f32, device=dev)

    @property
    def counters(self) -> torch.Tensor:
        """[T+1, 4] int32 record: per step total edge count (col 0) and overflow flag (col 1)."""
        if self.n_nets > 1:
            c = self._net_counters
            return torch.cat([c[:, :, :1].sum(dim=1, dtype=torch.int32), c[:, :, 1:].amax(dim=1)], dim=1)
        return self.chains[0].counters

    def net_counters(self, k: int) -> torch.Tensor:
        """[T+1, 4] int32 record of network k's environments (the engine's counters when n_nets = 1)."""
        return self._net_counters[:, k] if self.n_nets > 1 else self.chains[0].counters

    # ------------------------------------------------------------------ one env step (enqueue only)
    def _build(self, ch: _Chain, t: int, stream: int) -> None:
        env, d = self.env, ch.desc
        rc = env.lib.gcbf_graph_build(C.byref(d), self.agent[t, ch.e0].data_ptr(),
                                      self.obstacles[ch.e0].data_ptr() if self.O > 0 else None,
                                      env.ray_table.data_ptr(), self.hits[t, ch.e0].data_ptr(),
                                      ch.row_start[t % 2].data_ptr(), ch.row_deg[t % 2].data_ptr(),
                                      ch.edge_recv[t % 2].data_ptr(), ch.edge_src[t % 2].data_ptr(),
                                      ch.counters[t].data_ptr(), self._build_flags, stream)
        _lib.check(rc, "gcbf_graph_build")

    def _step(self, ch: _Chain, t: int, stream: int) -> None:
        env, d = self.env, ch.desc
        obs = self.obstacles[ch.e0].data_ptr() if self.O > 0 else None
        b = t % 2
        if self.policy == "actor_refine":
            self._step_refine(ch, t, stream)
            return
        if self.policy in QP_FILTER_POLICIES:
            self._step_qp_filter(ch, t, stream)
            return
        if self.policy == "actor":      # algo.step + env.step + get_graph(next) in one call
            rc = env.lib.gcbf_rollout_step_l(
                C.byref(d), self.n_layers, self.params_buf.data_ptr(), self.infer_blob.data_ptr(), self.use_tc,
                self.agent[t, ch.e0].data_ptr(), self.goal[ch.e0].data_ptr(), obs, env.ray_table.data_ptr(),
                self.hits[t, ch.e0].data_ptr(), ch.row_start[b].data_ptr(), ch.row_deg[b].data_ptr(),
                ch.edge_recv[b].data_ptr(), ch.edge_src[b].data_ptr(), ch.counters[t].data_ptr(),
                self.actions[t, ch.e0].data_ptr(), self.agent[t + 1, ch.e0].data_ptr(),
                self.hits[t + 1, ch.e0].data_ptr(), ch.row_start[1 - b].data_ptr(), ch.row_deg[1 - b].data_ptr(),
                ch.edge_recv[1 - b].data_ptr(), ch.edge_src[1 - b].data_ptr(), ch.counters[t + 1].data_ptr(),
                self.rewards[t, ch.e0:].data_ptr(), self.costs[t, ch.e0:].data_ptr(), ch.ws.data_ptr(), ch.ws.numel(),
                stream)
            _lib.check(rc, "gcbf_rollout_step_l")
            return
        mode = 2                        # u_ref policy
        if self.controller is not None:  # CBF-QP action, then env.step with it as input
            c = self.controller
            rc = getattr(env.lib, c._ENTRY)(C.byref(d), c.alpha, c.max_iter, c.tol, self.agent[t, ch.e0].data_ptr(),
                                            self.goal[ch.e0].data_ptr(), self.hits[t, ch.e0].data_ptr(),
                                            self.actions[t, ch.e0].data_ptr(), ch.qp_r.data_ptr(),
                                            ch.qp_iters[t].data_ptr(), ch.qp_ws.data_ptr(), ch.qp_ws.numel(), stream)
            _lib.check(rc, c._ENTRY)
            mode = env.action_step_mode
        rc = env.lib.gcbf_env_step(C.byref(d), self.agent[t, ch.e0].data_ptr(), self.goal[ch.e0].data_ptr(), obs,
                                   None, ch.row_start[b].data_ptr(), ch.row_deg[b].data_ptr(), ch.edge_src[b].data_ptr(),
                                   self.actions[t, ch.e0].data_ptr(), self.agent[t + 1, ch.e0].data_ptr(),
                                   self.rewards[t, ch.e0:].data_ptr(), self.costs[t, ch.e0:].data_ptr(), mode, stream)
        _lib.check(rc, "gcbf_env_step")
        self._build(ch, t + 1, stream)

    def _step_refine(self, ch: _Chain, t: int, stream: int) -> None:
        """policy forward -> refined action (gcbf_refine_actions, iterations recorded per graph) -> env.step with it as
        input -> graph build of the next state."""
        env, d = self.env, ch.desc
        if self.cbf_params is None:
            raise RuntimeError("the actor_refine policy needs the CBF: call set_cbf_params() before run()")
        b = t % 2
        args = (self.agent[t, ch.e0], self.goal[ch.e0], self.hits[t, ch.e0], ch.row_start[b], ch.row_deg[b],
                ch.edge_recv[b], ch.edge_src[b], ch.counters[t])
        rc = env.lib.gcbf_gnn_infer(C.byref(d), _lib.NET_ACTOR, env.action_dim, self.params_buf.data_ptr(),
                                    self.infer_blob.data_ptr(), self.use_tc, *[_lib.ptr(x) for x in args], 0,
                                    ch.pi.data_ptr(), ch.ws.data_ptr(), ch.ws.numel(), stream)
        _lib.check(rc, "gcbf_gnn_infer")
        launch_refine(env, d, self.refine_alpha, self.refine_lr, self.refine_max_iter, self.use_tc, self.cbf_params,
                      self._refine_planes, ch.pi, *args, self.actions[t, ch.e0], None,
                      ch.refine_iters[t], ch.refine_ws, stream)
        obs = self.obstacles[ch.e0].data_ptr() if self.O > 0 else None
        rc = env.lib.gcbf_env_step(C.byref(d), self.agent[t, ch.e0].data_ptr(), self.goal[ch.e0].data_ptr(), obs,
                                   None, ch.row_start[b].data_ptr(), ch.row_deg[b].data_ptr(), ch.edge_src[b].data_ptr(),
                                   self.actions[t, ch.e0].data_ptr(), self.agent[t + 1, ch.e0].data_ptr(),
                                   self.rewards[t, ch.e0:].data_ptr(), self.costs[t, ch.e0:].data_ptr(), 1, stream)
        _lib.check(rc, "gcbf_env_step")
        self._build(ch, t + 1, stream)

    def _step_qp_filter(self, ch: _Chain, t: int, stream: int) -> None:
        """nominal action (actor_qp: policy forward and 2 pi + u_ref; u_ref_qp: u_ref) -> the CBF-QP nearest to it
        (gcbf_qp_filter; iterations, nominal and (lam, r) recorded) -> env.step with the filtered action as input ->
        graph build of the next state."""
        env, d = self.env, ch.desc
        if self.cbf_params is None:
            raise RuntimeError(f"the {self.policy} policy needs the CBF: call set_cbf_params() before run()")
        b = t % 2
        args = (self.agent[t, ch.e0], self.goal[ch.e0], self.hits[t, ch.e0], ch.row_start[b], ch.row_deg[b],
                ch.edge_recv[b], ch.edge_src[b], ch.counters[t])
        pi = None
        if self.policy == "actor_qp":
            rc = env.lib.gcbf_gnn_infer(C.byref(d), _lib.NET_ACTOR, env.action_dim, self.params_buf.data_ptr(),
                                        self.infer_blob.data_ptr(), self.use_tc, *[_lib.ptr(x) for x in args], 0,
                                        ch.pi.data_ptr(), ch.ws.data_ptr(), ch.ws.numel(), stream)
            _lib.check(rc, "gcbf_gnn_infer")
            pi = ch.pi.data_ptr()
        nominal = ch.qp_nominal[t]
        _lib.check(env.lib.gcbf_act(C.byref(d), _lib.ptr(args[0]), _lib.ptr(args[1]), pi, nominal.data_ptr(), stream),
                   "gcbf_act")
        # u_ref_qp solves with u_nom = NULL: the kernel's own u_ref, the labels' QP (recorded above for the statistics)
        rc = env.lib.gcbf_qp_filter(C.byref(d), self.refine_alpha, self.use_tc, QP_MAX_ITER, QP_TOL,
                                    self.cbf_params.flat.data_ptr(), *[_lib.ptr(x) for x in args],
                                    nominal.data_ptr() if self.policy == "actor_qp" else None,
                                    self.actions[t, ch.e0].data_ptr(), ch.qp_aux[t].data_ptr(),
                                    ch.qp_iters[t].data_ptr(), ch.qp_ws.data_ptr(), ch.qp_ws.numel(), stream)
        _lib.check(rc, "gcbf_qp_filter")
        obs = self.obstacles[ch.e0].data_ptr() if self.O > 0 else None
        rc = env.lib.gcbf_env_step(C.byref(d), self.agent[t, ch.e0].data_ptr(), self.goal[ch.e0].data_ptr(), obs,
                                   None, ch.row_start[b].data_ptr(), ch.row_deg[b].data_ptr(), ch.edge_src[b].data_ptr(),
                                   self.actions[t, ch.e0].data_ptr(), self.agent[t + 1, ch.e0].data_ptr(),
                                   self.rewards[t, ch.e0:].data_ptr(), self.costs[t, ch.e0:].data_ptr(), 1, stream)
        _lib.check(rc, "gcbf_env_step")
        self._build(ch, t + 1, stream)

    def _enqueue_persistent(self, n_steps: int, stream: int) -> None:
        env, ch = self.env, self.chains[0]
        if self.n_nets > 1:
            rc = env.lib.gcbf_rollout_persistent_multi(
                C.byref(self._pdesc), int(n_steps), self.n_nets, self.params_buf.data_ptr(), self.infer_blob.data_ptr(),
                self._net_of_env.data_ptr(), self.goal.data_ptr(), self.obstacles.data_ptr() if self.O > 0 else None,
                env.ray_table.data_ptr(), self.agent.data_ptr(), self.hits.data_ptr(), self.actions.data_ptr(),
                self.rewards.data_ptr(), self.costs.data_ptr(), self._net_counters.data_ptr(), self._pws.data_ptr(),
                self._pws.numel(), self.phase_stamps.data_ptr() if self.phase_stamps is not None else None, stream)
            _lib.check(rc, "gcbf_rollout_persistent_multi")
            return
        rc = env.lib.gcbf_rollout_persistent(
            C.byref(self._pdesc), int(n_steps), self.params_buf.data_ptr(), self.infer_blob.data_ptr(), self.goal.data_ptr(),
            self.obstacles.data_ptr() if self.O > 0 else None, env.ray_table.data_ptr(), self.agent.data_ptr(),
            self.hits.data_ptr(), self.actions.data_ptr(), self.rewards.data_ptr(), self.costs.data_ptr(),
            ch.counters.data_ptr(), self._pws.data_ptr(), self._pws.numel(),
            self.phase_stamps.data_ptr() if self.phase_stamps is not None else None, stream)
        _lib.check(rc, "gcbf_rollout_persistent")

    def _enqueue_all(self) -> None:
        stream = torch.cuda.current_stream(self.env.device).cuda_stream
        if self.persistent:
            self._enqueue_persistent(self.T, stream)
            return
        ch = self.chains[0]
        self._build(ch, 0, stream)
        for t in range(self.T):
            self._step(ch, t, stream)

    # ------------------------------------------------------------------ public
    def set_initial(self, agent0: torch.Tensor, goal: torch.Tensor, obstacle) -> None:
        """Initial conditions: [E,N,sd] x2 (device or pinned host) + obstacle container."""
        self.agent[0].copy_(agent0.reshape(self.agent[0].shape), non_blocking=True)
        self.goal.copy_(goal.reshape(self.goal.shape), non_blocking=True)
        if self.O > 0:
            packed = obstacle.packed if hasattr(obstacle, "packed") else obstacle
            self.obstacles.copy_(packed.reshape(self.obstacles.shape), non_blocking=True)
        self._obstacle_obj = obstacle

    def _set_depth(self, n_layers: int) -> None:
        """Re-size the parameter / weight / workspace buffers for an actor with n_layers GNN layers.  The persistent
        kernel implements one layer, so a deeper actor runs on the step-by-step path; a one-layer actor gets the path
        the constructor chose for it, whatever actors the engine ran before."""
        env, dev, nu = self.env, self.env.device, self.env.action_dim
        if n_layers > 1 and self.policy == "actor_refine":
            raise NotImplementedError("online policy refinement implements gnn_layers = 1; the actor has %d GNN layers"
                                      % n_layers)
        if self.policy in QP_FILTER_POLICIES:
            require_one_layer(n_layers, f"the {self.policy} policy's actor")
        if n_layers > 1 and self._persistent_requested:
            raise ValueError("the persistent rollout implements one GNN layer; this actor has %d" % n_layers)
        if n_layers > 1 and not self.use_tc:
            raise ValueError("actors with more than one GNN layer run on the tensor-core path only "
                             "(GCBF_TENSOR_CORES=0 selects the strict-fp32 path, which implements one layer)")
        self.n_layers = n_layers
        self.persistent = self._persistent_one_layer and n_layers == 1
        if not self.persistent:
            self._pws = None
        elif self._pws is None:
            n = env.lib.gcbf_rollout_persistent_workspace_floats(C.byref(self._pdesc))
            self._pws = torch.empty(int(n), dtype=torch.float32, device=dev)
        self._graph = None
        self.params_buf = torch.zeros(_lib.param_count(env.edge_dim, nu, n_layers), dtype=torch.float32, device=dev)
        n_blob = env.lib.gcbf_infer_count(env.edge_dim, nu) if n_layers == 1 else \
            env.lib.gcbf_params_t_count_l(env.edge_dim, nu, n_layers)
        self.infer_blob = torch.zeros(int(n_blob), dtype=torch.float32, device=dev)
        ch = self.chains[0]
        ch.ws = torch.empty(int(env.lib.gcbf_rollout_workspace_floats_l(C.byref(ch.desc), n_layers)),
                            dtype=torch.float32, device=dev)

    def set_params(self, params) -> None:
        """The actor: one NetParams, or a list of n_nets of them (network k runs the environments net_envs[k]).  The
        parameters are COPIED: after they change, call set_params again."""
        if self.n_nets > 1:
            self._set_nets(check_nets(params, self.n_nets))
            return
        if not isinstance(params, NetParams):
            params = check_nets(params, 1)[0]
        if params.n_layers != self.n_layers:
            self._set_depth(params.n_layers)
        self.params_buf.copy_(params.flat, non_blocking=True)
        env = self.env
        if self.n_layers > 1:   # transposed tf32 planes of every layer's weights (gcbf_rollout_step_l's infer_blob)
            _lib.check(env.lib.gcbf_prepare_params_l(env.edge_dim, env.action_dim, self.n_layers,
                                                     _lib.ptr(self.params_buf), _lib.ptr(self.infer_blob),
                                                     env._stream()), "gcbf_prepare_params_l")
            return
        _lib.check(env.lib.gcbf_prepare_infer(env.edge_dim, env.action_dim, _lib.ptr(self.params_buf),
                                              _lib.ptr(self.infer_blob), env._stream()), "gcbf_prepare_infer")

    def _set_nets(self, nets: list) -> None:
        env = self.env
        depth = nets[0].n_layers
        if depth > 1 and self._persistent_requested:
            raise ValueError("the persistent rollout implements one GNN layer; these actors have %d" % depth)
        self.n_layers = depth
        self.persistent = self._multi_persistent and depth == 1
        if not self.persistent:        # one solo engine per network, run one after another
            if self._subs is None:
                self._subs = [RolloutEngine(env, len(idx), T=self.T, n_obs=self.O, use_cuda_graph=self.use_cuda_graph,
                                            policy=self.policy, persistent=self._persistent_arg)
                              for idx in self.net_envs]
            for sub, p in zip(self._subs, nets):
                sub.set_params(p)
            return
        # stacked flat parameters and one gcbf_prepare_infer per network into the stacked blob
        st = env._stream()
        for k, p in enumerate(nets):
            self.params_buf[k, :p.count].copy_(p.flat, non_blocking=True)
            _lib.check(env.lib.gcbf_prepare_infer(env.edge_dim, env.action_dim, _lib.ptr(self.params_buf[k]),
                                                  _lib.ptr(self.infer_blob[k]), st), "gcbf_prepare_infer")

    def _run_subs(self, check: bool) -> None:
        """Sequential path of several networks: network k's solo engine from its environments' initial conditions, then
        its record gathered into this engine's."""
        n = 0
        for k, (sub, idx) in enumerate(zip(self._subs, self.net_envs)):
            ix = torch.tensor(idx, dtype=torch.long, device=self.env.device)
            sub.set_initial(self.agent[0, ix], self.goal[ix], self.obstacles[ix] if self.O > 0 else None)
            sub.run(check=False)
            n += sub.launches_per_run
            for name in ("agent", "hits", "actions", "rewards", "costs"):
                getattr(self, name).index_copy_(1, ix, getattr(sub, name))
            self._net_counters[:, k].copy_(sub.counters)
        self.launches_per_run = n
        if check:
            self.check_overflow()

    def run(self, check: bool = True) -> None:
        """Run the T-step rollout from the current initial conditions (async)."""
        if self.n_nets > 1 and not self.persistent:
            if self._subs is None:
                raise RuntimeError("call set_params() before run()")
            self._run_subs(check)
            return
        dev = self.env.device
        ch = self.chains[0]
        counters = self._net_counters if self.n_nets > 1 else ch.counters
        counters.zero_()
        lib = self.env.lib
        if self.use_cuda_graph:
            if self._graph is None:
                # warm-up outside capture (lazy module load, function attributes)
                st = torch.cuda.current_stream(dev).cuda_stream
                if self.persistent:
                    self._enqueue_persistent(min(self.T, 1), st)
                    counters.zero_()
                else:
                    self._build(ch, 0, st)
                    self._step(ch, 0, st)
                torch.cuda.synchronize(dev)
                g = torch.cuda.CUDAGraph()
                n0 = lib.gcbf_launch_count()
                with torch.cuda.graph(g):
                    self._enqueue_all()
                self.launches_per_run = int(lib.gcbf_launch_count() - n0)
                self._graph = g
            self._graph.replay()
        else:
            n0 = lib.gcbf_launch_count()
            self._enqueue_all()
            self.launches_per_run = int(lib.gcbf_launch_count() - n0)
        if check:
            self.check_overflow()

    def set_cbf_params(self, params: NetParams, alpha: float = 1.0, lr: float = REFINE_LR,
                       max_iter: int = REFINE_MAX_ITER) -> None:
        """actor_refine: the CBF the actions are refined against and the refinement's alpha / step size / iteration
        cap.  actor_qp / u_ref_qp: the CBF of the safety filter and its alpha (lr and max_iter are the refinement's and
        unused; the QP runs with the labels' QP_MAX_ITER / QP_TOL).  The parameters are COPIED (like set_params):
        after they change, call set_cbf_params again."""
        qp = self.policy in QP_FILTER_POLICIES
        if self.policy != "actor_refine" and not qp:
            raise RuntimeError("set_cbf_params() is for the actor_refine, actor_qp and u_ref_qp policies")
        if qp:
            require_one_layer(params.n_layers, "the CBF-QP safety filter")
        else:
            require_one_layer_refine(params, "CBF")
        if int(max_iter) < 1:
            raise ValueError(f"max_iter must be >= 1, got {max_iter}")
        settings = (float(alpha), float(lr), int(max_iter))
        if self.cbf_params is None:
            self.cbf_params = params.clone()
            if not qp:
                self._refine_planes = planes_buffer(params)
        else:       # in place: a captured rollout keeps reading the same buffers
            self.cbf_params.flat.copy_(params.flat)
        if not qp:  # the QP filter builds the planes it needs itself, inside its launch sequence
            prepare_planes(self.cbf_params, self._refine_planes, self.use_tc,
                           torch.cuda.current_stream(self.env.device).cuda_stream)
        if settings != (self.refine_alpha, self.refine_lr, self.refine_max_iter):
            self._graph = None      # the settings are baked into the captured launches
        self.refine_alpha, self.refine_lr, self.refine_max_iter = settings

    def refine_stats(self) -> dict:
        """actor_refine: median / max refinement iterations and the graph-steps that stopped at the cap, over every
        graph-step of the last run() (reads the device record once; call after run())."""
        if self.policy != "actor_refine":
            raise RuntimeError("refine_stats() needs the actor_refine policy")
        st = iter_stats(self.chains[0].refine_iters.reshape(-1))
        st["graph_steps"] = st.pop("solves")
        return st

    def qp_stats(self) -> dict:
        """CBF-QP baselines and the actor_qp / u_ref_qp safety filters: median / max iterations and capped solves over
        every solve of the last run() (reads the device record once; call after run()).  The safety filters also report
        the mean |u - u_nom| over the agent-steps (`mean_correction`) and the fraction of agent-steps whose CBF
        condition was relaxed (r > 0, `relaxed_frac`); a solve counts as capped when it ran QP_MAX_ITER iterations."""
        ch = self.chains[0]
        if self.policy in QP_FILTER_POLICIES:
            st = iter_stats(ch.qp_iters, cap=QP_MAX_ITER)   # bit 30 marks the dense-graph path, not a cap
            st["mean_correction"] = float(torch.linalg.vector_norm(self.actions - ch.qp_nominal, dim=-1).mean())
            st["relaxed_frac"] = float((ch.qp_aux[..., 1] > 0).float().mean())
            return st
        if self.controller is None:
            raise RuntimeError("qp_stats() needs a CBF-QP baseline or safety-filter policy")
        return iter_stats(ch.qp_iters.reshape(-1))

    def check_overflow(self) -> None:
        c = self.counters.cpu()
        if int(c[:, 1].max()) != 0:
            cap = self._pdesc.edge_cap if self.persistent else self.desc.edge_cap
            raise RuntimeError(f"edge capacity overflow during rollout: up to {int(c[:, 0].max())} edges; edge_cap={cap}"
                               + (" split evenly over the environments / CTA pairs (persistent kernel)" if self.persistent
                                  else "") + "; raise env.edge_cap_per_agent")

    def result(self) -> Rollout:
        """trainer/data.py Rollout in the reference's (b, T) order (views/transposes of the record)."""
        dones = torch.zeros(self.E, self.T, dtype=torch.bool, device=self.env.device)
        return Rollout(agent=self.agent.transpose(0, 1), goal=self.goal, hits=self.hits.transpose(0, 1),
                       obstacle=self._obstacle_obj, actions=self.actions.transpose(0, 1),
                       rewards=self.rewards.transpose(0, 1), costs=self.costs.transpose(0, 1), dones=dones,
                       log_pis=None, n_edges=self.counters[:, 0])

    def net_result(self, k: int) -> Rollout:
        """result() restricted to network k's environments (net_envs[k], in environment order)."""
        if self.n_nets == 1:
            return self.result()
        ix = torch.tensor(self.net_envs[k], dtype=torch.long, device=self.env.device)
        ro = self.result()
        obs = self._obstacle_obj
        if obs is not None:
            obs = obs.select(ix.cpu().numpy()) if hasattr(obs, "select") else obs[ix]
        return Rollout(agent=ro.agent[ix], goal=ro.goal[ix], hits=ro.hits[ix], obstacle=obs, actions=ro.actions[ix],
                       rewards=ro.rewards[ix], costs=ro.costs[ix], dones=ro.dones[ix], log_pis=None,
                       n_edges=self._net_counters[:, k, 0])
