"""MultiAgentEnv -- host-side mirror of gcbfplus/env/base.py:34-269 over batched torch
tensors.  Every method that does arithmetic calls libgcbf_b200.so; tensors carry a
leading graph-batch dim G where the reference uses jax.vmap.

Not reproduced: the JAX threefry PRNG stream of `reset` (SURVEY 8f3) -- `reset(key)`
takes an int seed / numpy Generator and samples with NumPy (setup work, not timed).
"""
from __future__ import annotations

import ctypes as C
import math
from abc import ABC, abstractmethod
from typing import Callable, NamedTuple, Optional, Tuple

import numpy as np
import scipy.linalg
import torch

from .. import _lib
from ..utils import jrandom as jr
from ..utils.graph import SwarmGraph
from .obstacle import Rectangle, Sphere


class StepResult(NamedTuple):
    graph: SwarmGraph
    reward: torch.Tensor
    cost: torch.Tensor
    done: torch.Tensor
    info: dict


class RolloutResult(NamedTuple):
    """gcbfplus/env/base.py:27-33, compact: states instead of dense graphs."""
    Tp1_graph: dict          # {"agent": [T+1,G,N,sd], "goal": [G,N,sd], "hits": [T+1,G,N,R,pd], "obstacle": ...}
    T_action: torch.Tensor   # [T,G,N,nu]
    T_reward: torch.Tensor   # [T,G]
    T_cost: torch.Tensor     # [T,G]
    T_done: torch.Tensor     # [T,G]
    T_info: dict


def lqr(A: np.ndarray, B: np.ndarray, Q: np.ndarray, R: np.ndarray) -> np.ndarray:
    """gcbfplus/env/utils.py:24-46 (discrete-time LQR gain)."""
    X = scipy.linalg.solve_discrete_are(A, B, Q, R)
    return scipy.linalg.inv(B.T @ X @ B + R) @ (B.T @ X @ A)


def ray_table_2d(num_beams: int, sense_range: float) -> np.ndarray:
    """gcbfplus/env/utils.py:51-56: per-ray (cos, sin)(theta) * range, fp32, host-evaluated."""
    f = np.float32
    thetas = np.linspace(-np.pi, np.pi - 2 * np.pi / num_beams, num_beams).astype(f)
    rng = f(sense_range)
    return np.stack([np.cos(thetas).astype(f) * rng, np.sin(thetas).astype(f) * rng], axis=-1).astype(f)


def ray_table_3d(num_beams: int, sense_range: float) -> np.ndarray:
    """gcbfplus/env/utils.py:57-74: (n/2) x n (theta-major) directions + the two poles."""
    f = np.float32
    thetas = np.linspace(-np.pi / 2 + 2 * np.pi / num_beams, np.pi / 2 - 2 * np.pi / num_beams,
                         num_beams // 2).astype(f)
    phis = np.linspace(-np.pi, np.pi - 2 * np.pi / num_beams, num_beams).astype(f)
    rng = f(sense_range)
    ct, st = np.cos(thetas).astype(f), np.sin(thetas).astype(f)
    cp, sp = np.cos(phis).astype(f), np.sin(phis).astype(f)
    dx = (ct[:, None] * cp[None, :]) * rng
    dy = (ct[:, None] * sp[None, :]) * rng
    dz = np.broadcast_to((st * rng)[:, None], dx.shape)
    d = np.stack([dx, dy, dz], axis=-1).reshape(-1, 3)
    poles = np.array([[0, 0, rng], [0, 0, -rng]], dtype=f)
    return np.concatenate([d, poles], axis=0).astype(f)


class MultiAgentEnv(ABC):
    PARAMS: dict = {}
    ENV_ID: str = ""
    # state_dim, edge_dim, action_dim, pos_dim
    DIMS: Tuple[int, int, int, int] = (0, 0, 0, 0)

    def __init__(self, num_agents: int, area_size: float, max_step: int = 256, max_travel: float = None,
                 dt: float = 0.03, params: dict = None, device: str = "cuda"):
        self._num_agents = num_agents
        self._dt = dt
        self._params = self.PARAMS if params is None else params
        self._t = 0
        self._max_step = max_step
        self._max_travel = max_travel
        self._area_size = area_size
        self.device = torch.device(device)
        #: average edge budget per agent for the receiver-grouped edge lists (overflow is
        #: detected on the device and raised by SwarmGraph.check_overflow()).
        self.edge_cap_per_agent = 16
        self.host_reset = False   # True: sample start / goal positions with the NumPy restatement instead of the kernel
        self._K = None
        self._A = None
        self._B = None
        self._setup_dynamics()
        if self.pos_dim == 3:
            tab = ray_table_3d(self._params["n_rays"], self._params["comm_radius"])
        else:
            tab = ray_table_2d(self._params["n_rays"], self._params["comm_radius"])
        self._ray_table_np = tab
        self._ray_table = None
        self._lib = None

    # ------------------------------------------------------------------ properties
    @property
    def params(self) -> dict:
        return self._params

    @property
    def num_agents(self) -> int:
        return self._num_agents

    @property
    def max_travel(self) -> float:
        return self._max_travel

    @property
    def area_size(self) -> float:
        return self._area_size

    @property
    def dt(self) -> float:
        return self._dt

    @property
    def max_episode_steps(self) -> int:
        return self._max_step

    @property
    def state_dim(self) -> int:
        return self.DIMS[0]

    @property
    def node_dim(self) -> int:
        return 3

    @property
    def edge_dim(self) -> int:
        return self.DIMS[1]

    @property
    def action_dim(self) -> int:
        return self.DIMS[2]

    @property
    def pos_dim(self) -> int:
        return self.DIMS[3]

    @property
    def radius(self) -> float:
        return self._params.get("car_radius", self._params.get("drone_radius"))

    @property
    def n_rays_cast(self) -> int:
        return int(self._ray_table_np.shape[0])

    @property
    def n_hits(self) -> int:
        """Hit nodes kept per agent (2-D: min(n_rays, 32), env/utils.py:49; LinearDrone: 16)."""
        return min(self._params["n_rays"], 32)

    @property
    def lib(self):
        if self._lib is None:
            self._lib = _lib.load()
        return self._lib

    @property
    def ray_table(self) -> torch.Tensor:
        if self._ray_table is None:
            self._ray_table = torch.from_numpy(self._ray_table_np).to(self.device)
        return self._ray_table

    @abstractmethod
    def _setup_dynamics(self) -> None:
        pass

    @abstractmethod
    def state_lim(self, state=None):
        pass

    @abstractmethod
    def action_lim(self):
        pass

    # ------------------------------------------------------------------ descriptor
    def _thresholds(self) -> dict:
        """Env-specific label radii (SURVEY A.2).  Overridden by subclasses."""
        r = self.radius
        return dict(unsafe_agent=r * 2, unsafe_obs=r, safe_agent=r * 4, safe_obs=r * 2)

    def desc(self, n_graphs: int, n_obs: int, edge_cap: Optional[int] = None, obs_per_graph: int = 1) -> _lib.EnvDesc:
        d = _lib.EnvDesc()
        f = _lib.f32
        r = self.radius
        rc = self._params["comm_radius"]
        d.env_kind = _lib.ENV_KIND[self.ENV_ID]
        d.n_graphs, d.n_agents, d.n_obs = n_graphs, self.num_agents, n_obs
        d.n_rays, d.n_hits = self.n_rays_cast, self.n_hits
        d.edge_cap = int(edge_cap if edge_cap is not None else self.edge_cap(n_graphs))
        d.obs_per_graph = obs_per_graph
        d.comm_radius, d.comm_radius_p1, d.lidar_radius = f(rc), f(rc + 1), f(rc - 1e-1)
        d.dt, d.mass = f(self._dt), f(self._params.get("m", 1.0))
        d.radius, d.two_r, d.two_r_p1, d.half_r = f(r), f(r * 2), f(r * 2 + 1), f(r * 0.5)
        th = self._thresholds()
        d.unsafe_agent, d.unsafe_obs = f(th["unsafe_agent"]), f(th["unsafe_obs"])
        d.safe_agent, d.safe_obs = f(th["safe_agent"]), f(th["safe_obs"])
        d.warn_agent, d.warn_obs = f(3 * r), f(2 * r)
        d.four_r_sq, d.r_sq = f(4 * r ** 2), f(r ** 2)
        d.comm_sq_thr, d.lidar_sq_thr = _lib.sqrt_threshold(rc), _lib.sqrt_threshold(rc - 1e-1)
        lo, up = self.state_lim()
        fin = [float(v) for v in up if math.isfinite(float(v))]
        d.v_lim = f(fin[0]) if fin else float("inf")
        d.u_lim = f(float(self.action_lim()[1][0]))
        if self._K is not None:
            K = np.asarray(self._K, dtype=np.float32).reshape(-1)
            for i, v in enumerate(K):
                d.K[i] = float(v)
        if self._A is not None:
            for i, v in enumerate(np.asarray(self._A, dtype=np.float32).reshape(-1)):
                d.A[i] = float(v)
            for i, v in enumerate(np.asarray(self._B, dtype=np.float32).reshape(-1)):
                d.B[i] = float(v)
        return d

    def edge_cap(self, n_graphs: int) -> int:
        N = self.num_agents
        per_agent = min(self.edge_cap_per_agent, 1 + (N - 1) + self.n_hits)
        return max(int(n_graphs * N * per_agent), 64)

    def _stream(self) -> int:
        # the library launches on the CURRENT device with the stream handed in: make the env's device current so
        # that make_env(device="cuda:1") (or a rank whose LOCAL_RANK != 0) does not pair a device-1 stream with device 0
        idx = self.device.index if self.device.index is not None else torch.cuda.current_device()
        if torch.cuda.current_device() != idx:
            torch.cuda.set_device(idx)
        return torch.cuda.current_stream(self.device).cuda_stream

    def clip_state(self, state: torch.Tensor) -> torch.Tensor:
        lo, up = self.state_lim(state)
        return torch.minimum(torch.maximum(state, lo.to(state.device)), up.to(state.device))

    def clip_action(self, action: torch.Tensor) -> torch.Tensor:
        lo, up = self.action_lim()
        return torch.minimum(torch.maximum(action, lo.to(action.device)), up.to(action.device))

    # ------------------------------------------------------------------ obstacles / reset
    # The reference's reset draws from jax.random (threefry); utils/jrandom.py restates those draws on the host
    # so that a seed gives the reference's scenario (SURVEY f3).  Everything below is vectorised over the
    # environments (the reference vmaps reset over per-env keys, trainer/trainer.py:84-85,134-136).
    def _sample_obstacles(self, keys: np.ndarray):
        """double_integrator.py:86-101 (Rectangle) / linear_drone.py:95-104 (Sphere).
        keys [E, 2] -> (obstacles, keys' [E, 2]) with the reference's split order."""
        O, L = self._params["n_obs"], self.area_size
        lo, hi = self._params["obs_len_range"]
        k = jr.split(keys, 2)
        obstacle_key, key = k[:, 0], k[:, 1]
        if self.pos_dim == 2:
            pos = jr.uniform(obstacle_key, (O, 2), 0, L)
            k = jr.split(key, 2)
            length_key, key = k[:, 0], k[:, 1]
            ln = jr.uniform(length_key, (O, 2), lo, hi)
            k = jr.split(key, 2)
            theta_key, key = k[:, 0], k[:, 1]
            th = jr.uniform(theta_key, (O,), 0, 2 * np.pi)
            return Rectangle.create(pos, ln[..., 0], ln[..., 1], th, device=self.device), key
        pos = jr.uniform(obstacle_key, (O, 3), 0, L)
        k = jr.split(key, 2)
        r_key, key = k[:, 0], k[:, 1]
        rad = jr.uniform(r_key, (O,), lo / 2, hi / 2)
        return Sphere.create(pos, rad, device=self.device), key

    def _inside_np(self, pts: np.ndarray, packed: np.ndarray, r: float) -> np.ndarray:
        """Host restatement of inside_obstacles (env/obstacle.py:53-96,234-270) for reset's rejection sampling.
        pts [a, dim], packed [a, O, k] (one obstacle set per point) -> bool [a]."""
        if packed.shape[1] == 0:
            return np.zeros(pts.shape[0], dtype=bool)
        f = np.float32
        pts = pts.astype(f)
        r = f(r)
        if self.pos_dim == 3:
            d = np.sqrt(((pts[:, None, :] - packed[:, :, :3]) ** 2).sum(-1))
            return (d <= packed[:, :, 3] + r).any(axis=1)
        rel_x = pts[:, None, 0] - packed[:, :, 0]
        rel_y = pts[:, None, 1] - packed[:, :, 1]
        c, s = packed[:, :, 4], packed[:, :, 5]
        xx = np.abs(rel_x * c + rel_y * s) - packed[:, :, 2]
        yy = np.abs(rel_x * s - rel_y * c) - packed[:, :, 3]
        is_in = ((xx < r) & (yy < 0)) | ((xx < 0) & (yy < r)) | ((xx > 0) & (yy > 0) & (np.sqrt(xx ** 2 + yy ** 2) < r))
        return is_in.any(axis=1)

    def _sample_agents_goals(self, keys: np.ndarray, packed: np.ndarray):
        """gcbfplus/env/utils.py:134-226 get_node_goal_rng for E environments at once (keys [E, 2], packed
        [E, O, k]): sequential rejection sampling per agent with the reference's key chain -- split(this_key, 3) per
        agent, split(k, 2) per retry, the first goal candidate drawn in [0, max_travel) but retries in
        [-max_travel, max_travel), not-yet-placed agents/goals sitting at the origin, and a restart from agent 0
        (same key chain) when 1024 retries are exhausted."""
        E = keys.shape[0]
        n, dim, L = self.num_agents, self.pos_dim, self.area_size
        f = np.float32
        min_dist = f(4 * self.radius)
        max_iter = 1024
        mt = self._max_travel
        states = np.zeros((E, n, dim), dtype=f)
        goals = np.zeros((E, n, dim), dtype=f)
        agent_id = np.zeros(E, dtype=np.int64)
        this_key = np.array(keys, dtype=np.uint32)

        def dist_min(all_pts, p):
            return np.sqrt(((all_pts - p[:, None, :]) ** 2).sum(-1)).min(axis=1)

        while True:
            act = np.nonzero(agent_id < n)[0]
            if act.size == 0:
                return states, goals
            k3 = jr.split(this_key[act], 3)
            agent_key, goal_key = k3[:, 0], k3[:, 1]
            this_key[act] = k3[:, 2]
            pk = packed[act]
            # ---- agent position
            cand = jr.uniform(agent_key, (dim,), 0, L)
            it_a = np.zeros(act.size, dtype=np.int64)
            kk = agent_key.copy()
            st = states[act]
            while True:
                bad = ((dist_min(st, cand) <= min_dist) | self._inside_np(cand, pk, min_dist)) & (it_a < max_iter)
                idx = np.nonzero(bad)[0]
                if idx.size == 0:
                    break
                k2 = jr.split(kk[idx], 2)
                kk[idx] = k2[:, 1]
                it_a[idx] += 1
                cand[idx] = jr.uniform(k2[:, 0], (dim,), 0, L)
            states[act, agent_id[act]] = cand
            # ---- goal position
            if mt is None:
                g = jr.uniform(goal_key, (dim,), 0, L)
            else:
                g = jr.uniform(goal_key, (dim,), 0, mt) + cand
            it_g = np.zeros(act.size, dtype=np.int64)
            kk = goal_key.copy()
            gl = goals[act]
            while True:
                bad = (dist_min(gl, g) <= min_dist) | self._inside_np(g, pk, min_dist)
                bad |= (g < 0).any(axis=1) | (g > f(L)).any(axis=1)
                if mt is not None:
                    bad |= np.sqrt(((g - cand) ** 2).sum(-1)) > f(mt)
                bad &= it_g < max_iter
                idx = np.nonzero(bad)[0]
                if idx.size == 0:
                    break
                k2 = jr.split(kk[idx], 2)
                kk[idx] = k2[:, 1]
                it_g[idx] += 1
                if mt is None:
                    g[idx] = jr.uniform(k2[:, 0], (dim,), 0, L)
                else:
                    g[idx] = jr.uniform(k2[:, 0], (dim,), -mt, mt) + cand[idx]
            goals[act, agent_id[act]] = g
            agent_id[act] += 1
            fail = act[(it_a >= max_iter) | (it_g >= max_iter)]
            if fail.size:                                    # "if no solution is found, start over"
                agent_id[fail] = 0
                states[fail] = 0
                goals[fail] = 0

    def reset(self, key=0, n_envs: Optional[int] = None) -> SwarmGraph:
        """env.reset (double_integrator.py:83-112 and twins) for a batch of environments.
        key: per-env threefry keys uint32 [E, 2] (what the reference's vmapped reset receives); or a single key
        uint32 [2] / an int seed, expanded with split(key, n_envs) the way the trainer does (trainer.py:135)."""
        self._t = 0
        key = jr.as_key(key) if not isinstance(key, np.ndarray) else key.astype(np.uint32)
        if key.ndim == 1:
            keys = jr.split(key, int(n_envs or 1))
        else:
            keys = key
            assert n_envs is None or n_envs == keys.shape[0]
        E = keys.shape[0]
        obstacles, keys = self._sample_obstacles(keys)
        sd, pd = self.state_dim, self.pos_dim
        if torch.device(self.device).type == "cuda" and not self.host_reset:
            # device path: one warp per environment runs the reference's rejection sampler with the same key chain
            # (csrc/geometry.cu reset_kernel; the host sampler below is its cross-check, tests/test_gpu_reset.py)
            agent_t = torch.zeros(E, self.num_agents, sd, dtype=torch.float32, device=self.device)
            goal_t = torch.zeros_like(agent_t)
            keys_t = torch.from_numpy(np.ascontiguousarray(keys).view(np.int32)).to(self.device)
            d = self.desc(E, obstacles.n_obs, edge_cap=1)
            mt = -1.0 if self._max_travel is None else float(self._max_travel)
            rc = self.lib.gcbf_reset_positions_ex(C.byref(d), _lib.ptr(keys_t),
                                                  _lib.ptr(obstacles.packed) if obstacles.n_obs else None,
                                                  float(self.area_size), float(np.float32(4 * self.radius)), mt,
                                                  1 if jr.PARTITIONABLE else 0, _lib.ptr(agent_t), _lib.ptr(goal_t),
                                                  self._stream())
            _lib.check(rc, "gcbf_reset_positions")
            if type(self)._reset_extra is not MultiAgentEnv._reset_extra:      # DubinsCar headings (tiny, host)
                agent, goal = agent_t.cpu().numpy(), goal_t.cpu().numpy()
                self._reset_extra(keys, agent, goal)
                agent_t, goal_t = torch.from_numpy(agent).to(self.device), torch.from_numpy(goal).to(self.device)
            return self.get_graph(agent_t, goal_t, obstacles)
        packed = obstacles.packed.cpu().numpy()
        agent = np.zeros((E, self.num_agents, sd), dtype=np.float32)
        goal = np.zeros((E, self.num_agents, sd), dtype=np.float32)
        agent[:, :, :pd], goal[:, :, :pd] = self._sample_agents_goals(keys, packed)
        self._reset_extra(keys, agent, goal)
        return self.get_graph(torch.from_numpy(agent).to(self.device), torch.from_numpy(goal).to(self.device),
                              obstacles)

    def reset_np(self, key=0, n_envs: Optional[int] = None) -> SwarmGraph:
        return self.reset(key, n_envs)

    def _reset_extra(self, keys: np.ndarray, agent: np.ndarray, goal: np.ndarray) -> None:
        pass

    # ------------------------------------------------------------------ graph
    def get_graph(self, agent: torch.Tensor, goal: torch.Tensor, obstacle, hits: Optional[torch.Tensor] = None,
                  out: Optional[SwarmGraph] = None, edge_cap: Optional[int] = None) -> SwarmGraph:
        """env.get_graph (double_integrator.py:288-320): LiDAR + radius neighbour lists.
        With `hits` given only the topology is rebuilt (replayed graphs).  edge_cap overrides the
        edge_cap_per_agent sizing (callers that know an upper bound on the edge count)."""
        if agent.dim() == 2:
            agent, goal = agent[None], goal[None]
        agent = agent.contiguous().float()
        goal = goal.contiguous().float()
        G, N, _ = agent.shape
        assert N == self.num_agents
        O = obstacle.n_obs if obstacle is not None else 0
        per_graph = 1
        if obstacle is not None and obstacle.packed.shape[0] != G:
            assert obstacle.packed.shape[0] == 1, "obstacle batch must be G or 1"
            per_graph = 0
        d = self.desc(G, O, edge_cap=edge_cap, obs_per_graph=per_graph)
        dev = agent.device
        cast = hits is None
        if out is None:
            A = G * N
            if hits is None:
                hits = torch.empty(G, N, self.n_hits, self.pos_dim, device=dev, dtype=torch.float32)
            out = SwarmGraph(self, agent, goal, obstacle, hits.contiguous(),
                             torch.empty(A, dtype=torch.int32, device=dev), torch.empty(A, dtype=torch.int32, device=dev),
                             torch.zeros(d.edge_cap, dtype=torch.int32, device=dev),
                             torch.zeros(d.edge_cap, dtype=torch.int32, device=dev),
                             torch.zeros(4, dtype=torch.int32, device=dev))
        else:
            d.edge_cap = out.edge_recv.numel()
        obs_ptr = _lib.ptr(obstacle.packed) if O > 0 else None
        rc = self.lib.gcbf_graph_build(C.byref(d), _lib.ptr(out.agent), obs_ptr, _lib.ptr(self.ray_table),
                                       _lib.ptr(out.hits), _lib.ptr(out.row_start), _lib.ptr(out.row_deg),
                                       _lib.ptr(out.edge_recv), _lib.ptr(out.edge_src), _lib.ptr(out.counters),
                                       1 if cast else 0, self._stream())
        _lib.check(rc, "gcbf_graph_build")
        return out

    def add_edge_feats(self, graph: SwarmGraph, state: torch.Tensor) -> SwarmGraph:
        """double_integrator.py:275-286: same topology, all edge features recomputed from
        `state` ([G, 2N+NR, sd] or just the agent block [G, N, sd]) with the norm clip."""
        N = self.num_agents
        if state.dim() == 2:
            state = state[None]
        agent = state[:, :N].contiguous()
        return graph._replace(agent=agent, clip_all=True)

    # ------------------------------------------------------------------ control / step
    def u_ref(self, graph: SwarmGraph) -> torch.Tensor:
        """env.u_ref (double_integrator.py:332-338; dubins_car.py:328-379) -> [G, N, nu]."""
        G = graph.n_graphs
        d = self.desc(G, 0, edge_cap=graph.edge_recv.numel())
        out = torch.empty(G, self.num_agents, self.action_dim, device=graph.agent.device, dtype=torch.float32)
        _lib.check(self.lib.gcbf_act(C.byref(d), _lib.ptr(graph.agent), _lib.ptr(graph.goal), None, _lib.ptr(out),
                                     self._stream()), "gcbf_act")
        return out

    def _dynamics(self, graph: SwarmGraph, action: Optional[torch.Tensor], pi: Optional[torch.Tensor], mode: int):
        G, N = graph.n_graphs, self.num_agents
        O = graph.obstacle.n_obs if graph.obstacle is not None else 0
        per_graph = 0 if (graph.obstacle is not None and graph.obstacle.packed.shape[0] != G) else 1
        d = self.desc(G, O, edge_cap=graph.edge_recv.numel(), obs_per_graph=per_graph)
        dev = graph.agent.device
        if action is None:
            action = torch.empty(G, N, self.action_dim, device=dev, dtype=torch.float32)
        else:
            action = action.reshape(G, N, self.action_dim).contiguous().float()
        nxt = torch.empty_like(graph.agent)
        reward = torch.empty(G, device=dev, dtype=torch.float32)
        cost = torch.empty(G, device=dev, dtype=torch.float32)
        rc = self.lib.gcbf_env_step(C.byref(d), _lib.ptr(graph.agent), _lib.ptr(graph.goal),
                                    _lib.ptr(graph.obstacle.packed) if O > 0 else None, _lib.ptr(pi),
                                    _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_src),
                                    _lib.ptr(action), _lib.ptr(nxt), _lib.ptr(reward), _lib.ptr(cost), mode,
                                    self._stream())
        _lib.check(rc, "gcbf_env_step")
        return action, nxt, reward, cost

    def step(self, graph: SwarmGraph, action: torch.Tensor, get_eval_info: bool = False) -> StepResult:
        """env.step (double_integrator.py:145-181).  enable_stop = False (DubinsCar under DecShareCBF) steps without
        the stop mask (dubins_car.py:138-142)."""
        self._t += 1
        _, nxt, reward, cost = self._dynamics(graph, action, None, self.action_step_mode)
        done = torch.zeros(graph.n_graphs, dtype=torch.bool, device=graph.agent.device)
        info = {}
        if get_eval_info:
            info["inside_obstacles"] = self.inside_obstacles(graph)
        return StepResult(self.get_graph(nxt, graph.goal, graph.obstacle), reward, cost, done, info)

    @property
    def action_step_mode(self) -> int:
        """gcbf_env_step mode of a step with a given action: 1, or 3 when the DubinsCar stop mask is off."""
        return 1 if getattr(self, "enable_stop", True) else 3

    def forward_graph(self, graph: SwarmGraph, action: torch.Tensor) -> SwarmGraph:
        """env.forward_graph (double_integrator.py:340-354): next agent states on the same
        topology, hit nodes and goals frozen, edge features norm-clipped."""
        _, nxt, _, _ = self._dynamics(graph, action, None, 1)
        return graph._replace(agent=nxt, clip_all=True)

    # ------------------------------------------------------------------ masks
    def _masks(self, graph: SwarmGraph, which: str) -> torch.Tensor:
        G, N = graph.n_graphs, self.num_agents
        O = graph.obstacle.n_obs if graph.obstacle is not None else 0
        per_graph = 0 if (graph.obstacle is not None and graph.obstacle.packed.shape[0] != G) else 1
        d = self.desc(G, O, edge_cap=1, obs_per_graph=per_graph)
        out = torch.empty(G, N, dtype=torch.uint8, device=graph.agent.device)
        args = {k: None for k in ("unsafe", "collision", "finish", "safe")}
        args[which] = _lib.ptr(out)
        rc = self.lib.gcbf_masks(C.byref(d), _lib.ptr(graph.agent), _lib.ptr(graph.goal), _lib.ptr(graph.hits),
                                 _lib.ptr(graph.obstacle.packed) if O > 0 else None, args["unsafe"], args["collision"],
                                 args["finish"], args["safe"], self._stream())
        _lib.check(rc, "gcbf_masks")
        return out.bool()

    def safe_mask(self, graph: SwarmGraph) -> torch.Tensor:
        return self._masks(graph, "safe")

    def unsafe_mask(self, graph: SwarmGraph) -> torch.Tensor:
        return self._masks(graph, "unsafe")

    def collision_mask(self, graph: SwarmGraph) -> torch.Tensor:
        return self._masks(graph, "collision")

    def finish_mask(self, graph: SwarmGraph) -> torch.Tensor:
        return self._masks(graph, "finish")

    def inside_obstacles(self, graph: SwarmGraph) -> torch.Tensor:
        """inside_obstacles(agent_pos, obstacles, r=radius): the eval info of env.step
        (double_integrator.py:172-175), independent of agent-agent collisions.  Computed by the collision-mask
        kernel on single-agent graphs (no other agent to collide with -> only the obstacle term is left)."""
        G, N = graph.n_graphs, self.num_agents
        O = graph.obstacle.n_obs if graph.obstacle is not None else 0
        dev = graph.agent.device
        if O == 0:
            return torch.zeros(G, N, dtype=torch.bool, device=dev)
        shared = graph.obstacle.packed.shape[0] != G
        agent = graph.agent.reshape(G * N, 1, self.state_dim).contiguous()
        goal = graph.goal.reshape(G * N, 1, self.state_dim).contiguous()
        packed = graph.obstacle.packed
        if not shared:
            packed = packed[:, None].expand(G, N, *packed.shape[1:]).reshape(G * N, *packed.shape[1:]).contiguous()
        out = torch.empty(G * N, dtype=torch.uint8, device=dev)
        chunk = 32768                                       # grid.y limit of the mask kernel
        for lo in range(0, G * N, chunk):
            hi = min(G * N, lo + chunk)
            d = self.desc(hi - lo, O, edge_cap=1, obs_per_graph=0 if shared else 1)
            d.n_agents = 1
            rc = self.lib.gcbf_masks(C.byref(d), _lib.ptr(agent[lo:hi]), _lib.ptr(goal[lo:hi]), None,
                                     _lib.ptr(packed if shared else packed[lo:hi]), None, _lib.ptr(out[lo:hi]), None,
                                     None, self._stream())
            _lib.check(rc, "gcbf_masks")
        return out.reshape(G, N).bool()

    # ------------------------------------------------------------------ rollouts
    def rollout_fn(self, policy: Callable, rollout_length: int = None) -> Callable:
        """gcbfplus/env/base.py:173-189: returns fn(key, n_envs=1) -> RolloutResult."""
        T = rollout_length or self.max_episode_steps

        def fn(key=0, n_envs: int = 1) -> RolloutResult:
            graph = self.reset(key, n_envs)
            agents, hits, actions, rewards, costs = [graph.agent], [graph.hits], [], [], []
            for _ in range(T):
                action = policy(graph)
                graph, reward, cost, done, info = self.step(graph, action, get_eval_info=False)
                agents.append(graph.agent)
                hits.append(graph.hits)
                actions.append(action)
                rewards.append(reward)
                costs.append(cost)
            graph.check_overflow()
            g = {"agent": torch.stack(agents), "goal": graph.goal, "hits": torch.stack(hits),
                 "obstacle": graph.obstacle}
            dones = torch.zeros(T, n_envs, dtype=torch.bool, device=graph.agent.device)
            return RolloutResult(g, torch.stack(actions), torch.stack(rewards), torch.stack(costs), dones, {})

        return fn

    def rollout_fn_jitstep(self, policy: Callable, rollout_length: int = None, noedge: bool = False,
                           nograph: bool = False):
        """gcbfplus/env/base.py:191-259: same as rollout_fn plus per-step collision / finish masks."""
        T = rollout_length or self.max_episode_steps
        base = self.rollout_fn(policy, T)

        def fn(key=0, n_envs: int = 1):
            res = base(key, n_envs)
            unsafe, finish = self.rollout_masks(res)
            return res, unsafe.cpu().numpy(), finish.cpu().numpy()

        return fn

    def rollout_masks(self, res: RolloutResult):
        """test.py:147-148: collision / finish masks of every graph of a rollout -> [T+1, G, N]."""
        ag = res.Tp1_graph["agent"]
        Tp1, G, N, sd = ag.shape
        goal = res.Tp1_graph["goal"][None].expand(Tp1, G, N, sd).reshape(Tp1 * G, N, sd).contiguous()
        obs = res.Tp1_graph["obstacle"]
        rep = obs.repeat(Tp1)
        g = SwarmGraph(self, ag.reshape(Tp1 * G, N, sd).contiguous(), goal, rep,
                       res.Tp1_graph["hits"].reshape(Tp1 * G, N, self.n_hits, self.pos_dim).contiguous(),
                       None, None, torch.empty(1, dtype=torch.int32, device=ag.device), None, None)
        col = self._masks(g, "collision").reshape(Tp1, G, N)
        fin = self._masks(g, "finish").reshape(Tp1, G, N)
        return col, fin

    def render_video(self, *args, **kwargs) -> None:
        raise NotImplementedError("video rendering is out of scope of the CUDA hot path (SURVEY 2, row 17)")
