"""Batched closed-loop rollout -- replaces jit(vmap(rollout)) of gcbfplus/trainer/utils.py:25-55
and trainer/trainer.py:81-87.

Two device paths with the same arithmetic (bit-identical results, tests/test_gpu_rollout.py):
* persistent (default where supported: 2-D environments, n <= 512): ONE kernel launch for the whole T-step rollout, one
  thread-block cluster per environment looping over the steps (csrc/rollout_persist.cu);
* 5-launch env-step (gcbf_rollout_step), the whole T-step loop captured in one CUDA graph: LinearDrone, n > 512,
  GCBF_PERSISTENT=0, the u_ref policy, and actors with more than one GNN layer (gcbf_rollout_step_l; the engine takes
  the depth from the network set_params() receives).
No host sync inside the loop on either path.
The CBF-QP baselines (algo/cbf_qp.py) run on the CUDA-graph path: per step the pairwise CBFs + QP solve (2 launches),
env.step with the QP action as input, and the graph build of the next state.
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Optional

import torch

from .. import _lib
from ..algo.cbf_qp import BASELINES, iter_stats
from ..algo.params import NetParams
from ..utils.graph import SwarmGraph
from .data import Rollout


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
        # other half (gcbf_rollout_step's fused tail + graph build reads the old lists for the step cost)
        self.row_start = torch.zeros(2, E * N, dtype=i32, device=dev)
        self.row_deg = torch.zeros(2, E * N, dtype=i32, device=dev)
        self.edge_recv = torch.zeros(2, cap, dtype=i32, device=dev)
        self.edge_src = torch.zeros(2, cap, dtype=i32, device=dev)
        self.counters = torch.zeros(eng.T + 1, 4, dtype=i32, device=dev)
        n_ws = env.lib.gcbf_rollout_workspace_floats(C.byref(self.desc))
        self.ws = torch.empty(int(n_ws), dtype=f32, device=dev)
        if eng.controller is not None:
            # CBF-QP baseline: pairwise-CBF workspace, relaxations (scratch) and the per-step iteration record
            n_qp = env.lib.gcbf_cbfqp_workspace_floats(C.byref(self.desc))
            self.qp_ws = torch.empty(int(n_qp), dtype=f32, device=dev)
            self.qp_r = torch.empty(E, N, 3, dtype=f32, device=dev)
            self.qp_iters = torch.zeros(eng.T, eng.controller._n_solves(E, N), dtype=i32, device=dev)


class RolloutEngine:
    def __init__(self, env, n_envs: int, T: Optional[int] = None, n_obs: Optional[int] = None,
                 use_cuda_graph: bool = True, policy: str = "actor", persistent: Optional[bool] = None):
        """policy: 'actor' (a = 2 pi + u_ref, algo.step), 'u_ref' (test.py --u-ref), or a CBF-QP baseline: a
        DecShareCBF / CentralizedCBF object, or its name ('dec_share_cbf' / 'centralized_cbf': built with alpha = 1)."""
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
        elif policy not in ("actor", "u_ref"):
            raise ValueError(f"unknown rollout policy {policy!r}")
        if self.controller is None and not getattr(env, "enable_stop", True):
            raise ValueError("the actor / u_ref rollouts apply the DubinsCar stop mask; env.enable_stop is False "
                             "(set by DecShareCBF)")
        self.policy = policy
        self.use_cuda_graph = use_cuda_graph
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
        if persistent is None:
            # default only where every environment's cluster is resident at once (level 2): otherwise the environments
            # beyond the resident clusters run in a second round
            # DubinsCar is opt-in: its persistent rollout agrees with the 5-launch path only to closed-loop rounding.
            # States and actions are identical while every speed is 0
            # (step 0); from the first step with v != 0 a few policy outputs differ by 1-2 ulp (1.8e-7) -- the
            # (v cos th, v sin th) edge features are evaluated in two translation units -- which the closed loop
            # amplifies to 1.6e-5 after 24 steps.  Env-sharded runs must not mix two numeric paths.
            persistent = (level == 2 and env.ENV_ID != "DubinsCar" and os.environ.get("GCBF_PERSISTENT", "1") != "0")
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
        self._graph: Optional[torch.cuda.CUDAGraph] = None
        self.launches_per_run = 0
        self._obstacle_obj = None

    @property
    def counters(self) -> torch.Tensor:
        """[T+1, 4] int32 record: per step total edge count (col 0) and overflow flag (col 1)."""
        return self.chains[0].counters

    # ------------------------------------------------------------------ one env step (enqueue only)
    def _build(self, ch: _Chain, t: int, stream: int) -> None:
        env, d = self.env, ch.desc
        rc = env.lib.gcbf_graph_build(C.byref(d), self.agent[t, ch.e0].data_ptr(),
                                      self.obstacles[ch.e0].data_ptr() if self.O > 0 else None,
                                      env.ray_table.data_ptr(), self.hits[t, ch.e0].data_ptr(),
                                      ch.row_start[t % 2].data_ptr(), ch.row_deg[t % 2].data_ptr(),
                                      ch.edge_recv[t % 2].data_ptr(), ch.edge_src[t % 2].data_ptr(),
                                      ch.counters[t].data_ptr(), 1 | 8, stream)      # bit 3: rows in ticket order
        _lib.check(rc, "gcbf_graph_build")

    def _step(self, ch: _Chain, t: int, stream: int) -> None:
        env, d = self.env, ch.desc
        obs = self.obstacles[ch.e0].data_ptr() if self.O > 0 else None
        b = t % 2
        if self.policy == "actor" and self.n_layers > 1:
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
        if self.policy == "actor":      # algo.step + env.step + get_graph(next) in one call (6 launches)
            rc = env.lib.gcbf_rollout_step(
                C.byref(d), self.params_buf.data_ptr(), self.infer_blob.data_ptr(), self.use_tc,
                self.agent[t, ch.e0].data_ptr(), self.goal[ch.e0].data_ptr(), obs, env.ray_table.data_ptr(),
                self.hits[t, ch.e0].data_ptr(), ch.row_start[b].data_ptr(), ch.row_deg[b].data_ptr(),
                ch.edge_recv[b].data_ptr(), ch.edge_src[b].data_ptr(), ch.counters[t].data_ptr(),
                self.actions[t, ch.e0].data_ptr(), self.agent[t + 1, ch.e0].data_ptr(),
                self.hits[t + 1, ch.e0].data_ptr(), ch.row_start[1 - b].data_ptr(), ch.row_deg[1 - b].data_ptr(),
                ch.edge_recv[1 - b].data_ptr(), ch.edge_src[1 - b].data_ptr(), ch.counters[t + 1].data_ptr(),
                self.rewards[t, ch.e0:].data_ptr(), self.costs[t, ch.e0:].data_ptr(), ch.ws.data_ptr(), ch.ws.numel(),
                stream)
            _lib.check(rc, "gcbf_rollout_step")
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

    def _enqueue_persistent(self, n_steps: int, stream: int) -> None:
        env, ch = self.env, self.chains[0]
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

    def set_params(self, params: NetParams) -> None:
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

    def run(self, check: bool = True) -> None:
        """Run the T-step rollout from the current initial conditions (async)."""
        dev = self.env.device
        ch = self.chains[0]
        ch.counters.zero_()
        lib = self.env.lib
        if self.use_cuda_graph:
            if self._graph is None:
                # warm-up outside capture (lazy module load, function attributes)
                st = torch.cuda.current_stream(dev).cuda_stream
                if self.persistent:
                    self._enqueue_persistent(min(self.T, 1), st)
                    ch.counters.zero_()
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

    def qp_stats(self) -> dict:
        """CBF-QP baselines: median / max iterations and capped solves over every solve of the last run() (reads the
        device record once; call after run())."""
        if self.controller is None:
            raise RuntimeError("qp_stats() needs a CBF-QP baseline policy")
        return iter_stats(self.chains[0].qp_iters.reshape(-1))

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
