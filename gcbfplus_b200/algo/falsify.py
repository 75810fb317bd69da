"""Falsification of a trained GCBF+ CBF: gradient search over the agent states for violations of the CBF condition under
the policy (gcbf_cbf_condition on the device).

For one graph with states x, fixed goals and obstacles, a = 2 pi(g) + u_ref(x) and g' = forward_graph(g, a):
  term_i = -(h_i(g') - h_i(g)) / dt - alpha h_i(g),   J = max term_i over the agents with h_i(g) >= 0 and a finite term.
A counterexample is (x, i) with h_i(g) >= 0 and term_i > 0: an agent the CBF calls safe from which the closed loop the
rollout runs breaks the condition.  GCBFPlus.falsify climbs J per graph by normalised gradient steps (DESIGN 4.10)."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from .. import _lib
from .params import NetParams

FALSIFY_LR = 0.01


def require_one_layer_falsify(params: NetParams, what: str) -> None:
    """The state gradient runs on the one-layer data-only backward (as the refinement)."""
    if params.n_layers != 1:
        raise NotImplementedError(f"the CBF-condition gradient implements gnn_layers = 1; the {what} has "
                                  f"{params.n_layers} GNN layers")


def prepare_planes(params: NetParams, use_tc: int, stream: int) -> torch.Tensor:
    """gcbf_cbf_condition_prepare: the backward-data operands of the CURRENT parameters (tf32 planes on the tensor-core
    path, transposed weights on the strict-fp32 path)."""
    lib = _lib.load()
    n = int(lib.gcbf_params_t_count_l(params.edge_dim, params.out_dim, 1))
    planes = torch.empty(n, dtype=torch.float32, device=params.flat.device)
    _lib.check(lib.gcbf_cbf_condition_prepare(params.edge_dim, params.out_dim, int(use_tc), _lib.ptr(params.flat),
                                              _lib.ptr(planes), n, stream), "gcbf_cbf_condition_prepare")
    return planes


class CbfCondition:
    """The two networks' planes (built once: the parameters must not change while it is used) and the workspace of
    the last batch shape."""

    def __init__(self, algo, actor: Optional[NetParams] = None):
        self.algo = algo
        self.env = algo._env
        self.cbf = algo.cbf_params
        self.actor = actor or algo.actor_net_params
        require_one_layer_falsify(self.cbf, "CBF")
        require_one_layer_falsify(self.actor, "actor")
        self.use_tc = 1 if _lib.USE_TC else 0
        stream = self.env._stream()
        self.cbf_planes = prepare_planes(self.cbf, self.use_tc, stream)
        self.actor_planes = prepare_planes(self.actor, self.use_tc, stream)
        self._ws: Optional[torch.Tensor] = None
        self._ws_key = None

    def __call__(self, graph, with_grad: bool = False):
        """(h [G, N], term [G, N], worst [G] int32[, grad [G, N, sd]])."""
        env = self.env
        G, N = graph.n_graphs, env.num_agents
        d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
        if self._ws_key != (G, d.edge_cap):
            self._ws = None
            n = env.lib.gcbf_cbf_condition_workspace_floats(C.byref(d))
            if n <= 0:
                raise RuntimeError("gcbf_cbf_condition_workspace_floats: bad descriptor")
            self._ws = torch.empty(int(n), dtype=torch.float32, device=env.device)
            self._ws_key = (G, d.edge_cap)
        dev = graph.agent.device
        h = torch.empty(G, N, dtype=torch.float32, device=dev)
        term = torch.empty(G, N, dtype=torch.float32, device=dev)
        worst = torch.empty(G, dtype=torch.int32, device=dev)
        grad = torch.empty_like(graph.agent) if with_grad else None
        rc = env.lib.gcbf_cbf_condition(
            C.byref(d), float(self.algo.alpha), self.use_tc, _lib.ptr(self.cbf.flat), _lib.ptr(self.cbf_planes),
            _lib.ptr(self.actor.flat), _lib.ptr(self.actor_planes), _lib.ptr(graph.agent), _lib.ptr(graph.goal),
            _lib.ptr(graph.hits), _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_recv),
            _lib.ptr(graph.edge_src), _lib.ptr(graph.counters), _lib.ptr(h), _lib.ptr(term), _lib.ptr(worst),
            _lib.ptr(grad), _lib.ptr(self._ws), self._ws.numel(), env._stream())
        _lib.check(rc, "gcbf_cbf_condition")
        return (h, term, worst, grad) if with_grad else (h, term, worst)


def worst_value(term: torch.Tensor, worst: torch.Tensor) -> torch.Tensor:
    """J per graph: term of the worst agent, -inf where there is none."""
    idx = worst.long().clamp_min(0)
    j = term.gather(1, idx[:, None]).squeeze(1)
    return torch.where(worst >= 0, j, torch.full_like(j, -float("inf")))


def falsify(algo, agent: torch.Tensor, goal: torch.Tensor, obstacle, n_iter: int, lr: float = FALSIFY_LR,
            agents_per_chunk: int = 32768) -> dict:
    """Projected gradient ascent on J per graph from the states `agent` [G, N, sd] (goals [G, N, sd] and the obstacles
    fixed).  Iteration k rebuilds the graph at x_k, evaluates h, term, J and grad J, keeps the best J, and (k < n_iter
    - 1) steps x_{k+1} = clip_state(x_k + lr grad / |grad|) per graph; a graph with a zero gradient stays where it is.
    Graphs are processed in chunks of agents_per_chunk agents; an edge-capacity overflow doubles
    env.edge_cap_per_agent and runs the chunk again.

    Returns a dict of per-graph tensors: J0 (J at the start), J (the best J), worst (its agent), iter (its iteration),
    agent (its states), h / term ([G, N] at those states), and the false-safe counts false_safe0 / false_safe: agents
    with env.unsafe_mask set and h >= 0 at the start and at the best states."""
    if int(n_iter) < 1:
        raise ValueError(f"n_iter must be >= 1, got {n_iter}")
    env = algo._env
    cond = CbfCondition(algo)
    G, N = agent.shape[0], env.num_agents
    agent = agent.contiguous().float()
    goal = goal.contiguous().float()
    chunk = max(1, agents_per_chunk // N)
    out = {"J0": torch.empty(G, device=env.device), "J": torch.empty(G, device=env.device),
           "worst": torch.empty(G, dtype=torch.int32, device=env.device),
           "iter": torch.empty(G, dtype=torch.int32, device=env.device),
           "agent": torch.empty_like(agent), "h": torch.empty(G, N, device=env.device),
           "term": torch.empty(G, N, device=env.device)}
    fs0 = fs = 0
    for lo in range(0, G, chunk):
        hi = min(G, lo + chunk)
        obs = obstacle.select(slice(lo, hi)) if obstacle is not None and obstacle.packed.shape[0] == G else obstacle
        for _ in range(6):
            res = _falsify_chunk(env, cond, agent[lo:hi], goal[lo:hi], obs, int(n_iter), float(lr))
            if res is not None:
                break
            env.edge_cap_per_agent *= 2                  # rows were dropped: grow the edge lists and search again
        else:
            raise RuntimeError("edge capacity overflow persists after growing env.edge_cap_per_agent 64x")
        for k in out:
            out[k][lo:hi] = res[k]
        fs0 += res["false_safe0"]
        fs += res["false_safe"]
    out["false_safe0"], out["false_safe"] = fs0, fs
    return out


def _false_safe(env, graph, h) -> int:
    return int((env.unsafe_mask(graph) & (h >= 0)).sum().item())


def _falsify_chunk(env, cond: CbfCondition, x0, goal, obs, n_iter: int, lr: float) -> Optional[dict]:
    x = x0.clone()
    flag = torch.zeros(1, dtype=torch.int32, device=x.device)
    best = None
    for k in range(n_iter):
        graph = env.get_graph(x, goal, obs)
        flag |= graph.counters[1:2]
        h, term, worst, grad = cond(graph, with_grad=True)
        J = worst_value(term, worst)
        if best is None:
            best = {"J0": J.clone(), "J": J.clone(), "worst": worst.clone(), "agent": x.clone(), "h": h.clone(),
                    "term": term.clone(), "iter": torch.zeros_like(worst),
                    "false_safe0": _false_safe(env, graph, h)}
        else:
            up = J > best["J"]
            best["J"] = torch.where(up, J, best["J"])
            best["worst"] = torch.where(up, worst, best["worst"])
            best["iter"] = torch.where(up, torch.full_like(worst, k), best["iter"])
            best["agent"] = torch.where(up[:, None, None], x, best["agent"])
            best["h"] = torch.where(up[:, None], h, best["h"])
            best["term"] = torch.where(up[:, None], term, best["term"])
        if k + 1 < n_iter:
            # NaN rows (an agent at its goal) do not move the graph; a graph without a worst agent has grad 0
            g = torch.nan_to_num(grad, nan=0.0)
            nrm = g.flatten(1).norm(dim=1)
            step = torch.where(nrm > 0, lr / nrm, torch.zeros_like(nrm))
            x = env.clip_state(x + step[:, None, None] * g).contiguous()
    if int(flag.item()) != 0:
        return None
    gb = env.get_graph(best["agent"], goal, obs)
    best["false_safe"] = _false_safe(env, gb, best["h"])
    return best
