"""Oracle CBF condition under the policy and its state gradient (TEST INFRASTRUCTURE ONLY): the definitions of
gcbf_cbf_condition / GCBFPlus.falsify (DESIGN 4.10) restated on oracle.envs and oracle.nn, differentiated by
torch.autograd in the dtype of the oracle environment and parameters.

The topology and the LiDAR hit points are those of one sparse oracle graph `g`, held fixed: the edge features are
rebuilt from the agent states x as the device builds them (es(receiver) - es(sender); on g the goal edges norm-clipped,
on g' = forward_graph(g, a) every edge).  torch's relu differentiates as 1[x > 0], clip_action / clip_state
(torch.minimum / maximum against the limits) pass no gradient outside their limits."""
from __future__ import annotations

from dataclasses import replace

import torch

from oracle.envs import Graph, OracleEnv
from oracle.nn import net_forward


def features(env: OracleEnv, g: Graph, x: torch.Tensor, clip_all: bool) -> torch.Tensor:
    """Edge features of g's edges with the agent states x (goals and hits from g)."""
    N = env.num_agents
    es = env.edge_state(torch.cat([x, g.states[N:-1]], 0))
    f = es[g.receivers] - es[g.senders]
    if clip_all:
        return env._clip_pos(f)
    goal_edge = ((g.senders >= N) & (g.senders < 2 * N))[:, None]
    return torch.where(goal_edge, env._clip_pos(f), f)


def condition(env: OracleEnv, cbf_p, actor_p, g: Graph, x: torch.Tensor, alpha: float):
    """h, term [N] and x' as functions of x: a = 2 pi(g) + u_ref(x), x' = Euler(x, clip_action(a)),
    term = -(h(g') - h(g)) / dt - alpha h(g); NaN where x' is NaN."""
    N = env.num_agents
    goal = g.states[N:2 * N]
    ge = replace(g, edges=features(env, g, x, False))
    h = net_forward(cbf_p, ge, "cbf").squeeze(-1)
    a = 2 * net_forward(actor_p, ge, "actor") + env.u_ref(x, goal)
    xn = env.agent_step_euler(x, env.clip_action(a), goal)
    hn = net_forward(cbf_p, replace(g, edges=features(env, g, xn, True)), "cbf").squeeze(-1)
    term = -((hn - h) / env.dt) - alpha * h
    term = torch.where(torch.isnan(xn).any(dim=1), torch.full_like(term, float("nan")), term)
    return h, term, xn


def worst_agent(h: torch.Tensor, term: torch.Tensor) -> int:
    """argmax of term over the agents with h >= 0 and a finite term (first on ties), -1 where there is none."""
    ok = (h >= 0) & torch.isfinite(term)
    if not bool(ok.any()):
        return -1
    return int(torch.argmax(torch.where(ok, term, torch.full_like(term, -float("inf")))))


def objective(env, cbf_p, actor_p, g, x, alpha, agent=None) -> dict:
    """h, term, worst and J = term[worst] at x, and grad_x J (autograd).  agent: differentiate term[agent] instead of
    the worst agent's term (the finite-difference check picks its agent itself)."""
    xv = x.detach().clone().requires_grad_(True)
    h, term, _ = condition(env, cbf_p, actor_p, g, xv, alpha)
    w = worst_agent(h.detach(), term.detach())
    i = w if agent is None else agent
    out = {"h": h.detach(), "term": term.detach(), "worst": w}
    if i < 0:
        out["J"] = -float("inf")
        out["grad"] = torch.zeros_like(x)
        return out
    (grad,) = torch.autograd.grad(term[i], xv)
    out["J"] = float(term[i].detach())
    out["grad"] = grad
    return out


def term_at(env, cbf_p, actor_p, g, x, alpha, agent: int) -> float:
    with torch.no_grad():
        return float(condition(env, cbf_p, actor_p, g, x, alpha)[1][agent])
