"""Oracle of the CBF-QP baselines (TEST INFRASTRUCTURE ONLY -- never imported by the product).

One-graph restatement, in the reference's operation order, of the pairwise CBFs (gcbfplus/algo/utils.py:44-349,
k = 3) and of DecShareCBF / CentralizedCBF.get_qp_action (algo/dec_share_cbf.py:61-150, centralized_cbf.py:64-117).
The Jacobian comes from torch.func.jacfwd (like the reference's jax.jacfwd), not from the hand-derived formulas of
csrc/cbfqp.cu, so that it checks them.  The QPs are handed to oracle/qp.py's float64 tools (`kkt_residual`,
`solve_qp_slsqp`) in their [rows, cols] form; `solve_dual_batched` is the same accelerated dual ascent as
`oracle.qp.solve_qp_dual`, vectorised over a batch of problems (one per agent for DecShareCBF) and sparse-friendly
(CentralizedCBF at scale).
"""
from __future__ import annotations

from typing import Callable, Dict, Optional

import numpy as np
import scipy.sparse as sp
import torch

from oracle.envs import Graph, OracleEnv
from oracle.qp import RELAX_PENALTY, RELAX_WEIGHT, control_affine_dyn

K = 3
SELF_DIST = 1e2
GAIN = {"DoubleIntegrator": 10.0, "DubinsCar": 5.0, "LinearDrone": 3.0}


def h_offset(env: OracleEnv) -> float:
    """4 (1.01 r)^2 (SingleIntegrator, LinearDrone) or 4 r^2 (DoubleIntegrator, DubinsCar), a python float."""
    r = env.r
    return 4 * (1.01 * r) ** 2 if env.env_id in ("SingleIntegrator", "LinearDrone") else 4 * r ** 2


def hit_states(env: OracleEnv, g: Graph) -> torch.Tensor:
    """[N, R, sd] hit-node states ([hit_pos, 0...]) of a graph."""
    N = env.num_agents
    return g.states[2 * N:2 * N + N * g.n_hits].reshape(N, g.n_hits, -1)


def _vel(env: OracleEnv, x: torch.Tensor) -> torch.Tensor:
    pd = env.pos_dim
    if env.env_id == "DubinsCar":
        return x[..., 3:4] * torch.stack([torch.cos(x[..., 2]), torch.sin(x[..., 2])], dim=-1)
    return x[..., pd:2 * pd]


def _dist_sq(env: OracleEnv, agent: torch.Tensor, hits: torch.Tensor) -> torch.Tensor:
    """[N, N + R] squared distances to [agents | own hits], self entry = 100 (the kernel's operation order)."""
    N, pd = agent.shape[0], env.pos_dim
    pos_c = torch.cat([agent[None, :, :pd].expand(N, N, pd), hits[:, :, :pd]], dim=1)
    d = agent[:, None, :pd] - pos_c
    sq = d * d
    s = sq[..., 0] + sq[..., 1]
    if pd == 3:
        s = s + sq[..., 2]
    eye = torch.zeros_like(s, dtype=torch.bool)
    eye[:, :N] = torch.eye(N, dtype=torch.bool)
    return torch.where(eye, torch.full_like(s, SELF_DIST), s), pos_c


def k_nearest(env: OracleEnv, agent: torch.Tensor, hits: torch.Tensor):
    """(idx [N, 3] int64 (stable argsort: ties -> lower index), isobs [N, 3] bool)."""
    s, _ = _dist_sq(env, agent, hits)
    idx = torch.argsort(s, dim=1, stable=True)[:, :K]
    return idx, idx >= agent.shape[0]


def pairwise_h(env: OracleEnv, agent: torch.Tensor, hits: torch.Tensor, idx: torch.Tensor) -> torch.Tensor:
    """h [N, 3] for FIXED picks idx (differentiable in `agent`; hits are constants)."""
    N, pd = agent.shape[0], env.pos_dim
    s, pos_c = _dist_sq(env, agent, hits)
    rows = torch.arange(N)[:, None]
    h0 = s[rows, idx] - torch.tensor(h_offset(env), dtype=agent.dtype)
    if env.env_id == "SingleIntegrator":
        return h0
    vel_i = _vel(env, agent)
    vel_c = torch.cat([vel_i[None].expand(N, N, pd), torch.zeros(N, hits.shape[1], pd, dtype=agent.dtype)], dim=1)
    xdiff = agent[:, None, :pd] - pos_c[rows, idx]
    vdiff = vel_i[:, None, :] - vel_c[rows, idx]
    p = xdiff * vdiff
    dot = p[..., 0] + p[..., 1]
    if pd == 3:
        dot = dot + p[..., 2]
    return 2 * dot + GAIN[env.env_id] * h0


def pairwise(env: OracleEnv, agent: torch.Tensor, hits: torch.Tensor) -> Dict[str, torch.Tensor]:
    """Pairwise CBFs and the Lie terms of their jacfwd Jacobian wrt all agent states (working dtype of `agent`):
    idx, isobs, h, lf_h [N, 3]; hx [N, 3, N, sd]; lg [N, 3, N, nu]; lg_self / lg_other [N, 3, nu]."""
    N = agent.shape[0]
    idx, isobs = k_nearest(env, agent, hits)
    h = pairwise_h(env, agent, hits, idx)
    hx = torch.func.jacfwd(lambda x: pairwise_h(env, x, hits, idx))(agent)
    f, gm = control_affine_dyn(env, agent)
    lf = torch.einsum("ikjx,jx->ik", hx, f)
    lg = torch.einsum("ikjx,jxu->ikju", hx, gm)
    ar = torch.arange(N)
    lg_self = lg[ar, :, ar]                                       # [N, 3, nu]
    other = torch.where((idx < N) & (idx != ar[:, None]), idx, ar[:, None])
    lg_other = lg[ar[:, None], torch.arange(K)[None, :], other]   # [N, 3, nu]
    lg_other = torch.where(((idx < N) & (idx != ar[:, None]))[..., None], lg_other, torch.zeros_like(lg_other))
    return {"idx": idx, "isobs": isobs, "h": h, "lf_h": lf, "hx": hx, "lg": lg, "lg_self": lg_self,
            "lg_other": lg_other}


# ------------------------------------------------------------------------------------------------------ QP data
def dec_share_data(p: Dict, u_ref: torch.Tensor, alpha: float = 1.0) -> Dict[str, np.ndarray]:
    """DecShareCBF: per agent Lg [N, 3, nu] (own block), b [N, 3] = resp (Lf_h + alpha h), u_ref [N, nu]."""
    resp = torch.where(p["isobs"], torch.tensor(1.0, dtype=p["h"].dtype), torch.tensor(0.5, dtype=p["h"].dtype))
    b = resp * (p["lf_h"] + alpha * p["h"])
    to = lambda t: t.detach().to(torch.float64).numpy()
    return {"Lg": to(p["lg_self"]), "b": to(b), "u_ref": to(u_ref)}


def central_data(p: Dict, u_ref: torch.Tensor, alpha: float = 1.0) -> Dict[str, np.ndarray]:
    """CentralizedCBF: Lg [3N, N nu], b [3N] = Lf_h + alpha h, u_ref [N nu]."""
    N = p["h"].shape[0]
    b = p["lf_h"] + alpha * p["h"]
    to = lambda t: t.detach().to(torch.float64).numpy()
    return {"Lg": to(p["lg"]).reshape(N * K, -1), "b": to(b).reshape(-1), "u_ref": to(u_ref).reshape(-1)}


def central_from_blocks(idx: np.ndarray, lg_self: np.ndarray, lg_other: np.ndarray) -> sp.csr_matrix:
    """Sparse [3N, N nu] CentralizedCBF matrix from per-row blocks (the kernel's storage)."""
    N, _, nu = lg_self.shape
    rows, cols, vals = [], [], []
    for i in range(N):
        for k in range(K):
            r = i * K + k
            rows += [r] * nu
            cols += list(range(i * nu, (i + 1) * nu))
            vals += list(lg_self[i, k])
            j = int(idx[i, k])
            if j < N and j != i:
                rows += [r] * nu
                cols += list(range(j * nu, (j + 1) * nu))
                vals += list(lg_other[i, k])
    return sp.csr_matrix((np.asarray(vals, np.float64), (rows, cols)), shape=(N * K, N * nu))


def _primal(Lg, lam, u_ref, u_lim):
    if sp.issparse(Lg):
        v = u_ref + Lg.T @ lam
    else:
        v = u_ref + np.einsum("bkc,bk->bc", Lg, lam)
    u = np.clip(v, -u_lim, u_lim)
    return np.where(np.isnan(u_ref), np.nan, u), np.maximum(0.0, (lam - RELAX_PENALTY) / RELAX_WEIGHT)


def solve_dual_batched(Lg, b: np.ndarray, u_ref: np.ndarray, u_lim: float, *, tol: float = 1e-11,
                       max_iter: int = 400000):
    """oracle.qp.solve_qp_dual (row-scaled FISTA with gradient restart, float64) for a batch of problems.
    Dense: Lg [B, M, nu], b [B, M], u_ref [B, nu].  Sparse: Lg a scipy matrix [M, n], b [M], u_ref [n] (one problem).
    Returns (u, r, lam, iterations [B])."""
    sparse = sp.issparse(Lg)
    if sparse:
        Lg = sp.csr_matrix(Lg, dtype=np.float64)
        s = 1.0 / np.sqrt(np.asarray(Lg.multiply(Lg).sum(1)).ravel() + 1.0 / RELAX_WEIGHT)
        Ls = sp.diags(s) @ Lg
        sig = sp.linalg.svds(Ls, k=1, return_singular_vectors=False)[0] if min(Ls.shape) > 1 else abs(Ls).max()
        lip = np.array([sig ** 2 * 1.0001 + (s * s).max() / RELAX_WEIGHT])
        s, b, u_ref = s[None], b[None], u_ref
    else:
        s = 1.0 / np.sqrt((Lg * Lg).sum(-1) + 1.0 / RELAX_WEIGHT)
        lip = np.linalg.norm(Lg * s[..., None], 2, axis=(1, 2)) ** 2 + (s * s).max(1) / RELAX_WEIGHT
    B = s.shape[0]
    step = (1.0 / lip)[:, None]
    mu = np.zeros_like(s)
    y = mu.copy()
    t = np.ones(B)
    active = np.ones(B, dtype=bool)
    its = np.zeros(B, dtype=np.int64)

    def lg_u(u):
        return (Lg @ u)[None] if sparse else np.einsum("bkc,bc->bk", Lg, u)

    def primal(lam):
        return _primal(Lg, lam[0] if sparse else lam, u_ref, u_lim)

    for _ in range(max_iter):
        lam = s * y
        u, r = primal(lam)
        u = np.nan_to_num(u)   # a NaN u_ref component (agent exactly at its goal) does not steer the other components
        grad = s * (-lg_u(u) - (r[None] if sparse else r) - b)
        mn = np.maximum(0.0, y + step * grad)
        res = np.abs(mn - y).max(1) / step[:, 0]
        restart = (grad * (mn - mu)).sum(1) < 0
        t_new = np.where(restart, 1.0, 0.5 * (1 + np.sqrt(1 + 4 * t * t)))
        beta = np.where(restart, 0.0, (t - 1) / t_new)
        y_new = mn + beta[:, None] * (mn - mu)
        y[active], mu[active], t[active] = y_new[active], mn[active], t_new[active]
        its[active] += 1
        active &= ~(res < tol)
        if not active.any():
            break
    lam = s * mu
    u, r = primal(lam)
    if sparse:
        lam = lam[0]
    return u, r, lam, its


def solve_dec_share(d: Dict[str, np.ndarray], u_lim: float, **kw):
    return solve_dual_batched(d["Lg"], d["b"], d["u_ref"], u_lim, **kw)


def solve_central(d: Dict[str, np.ndarray], u_lim: float, **kw):
    return solve_dual_batched(sp.csr_matrix(d["Lg"]), d["b"], d["u_ref"], u_lim, **kw)


# ------------------------------------------------------------------------------------------------------ controllers
def act(env: OracleEnv, g: Graph, algo: str, alpha: float = 1.0) -> torch.Tensor:
    """DecShareCBF / CentralizedCBF.act on one graph: pairwise data in the working dtype, exact float64 QP ->
    action [N, nu] in the working dtype."""
    p = pairwise(env, g.agent, hit_states(env, g))
    ur = env.u_ref(g.agent, g.goal)
    u_lim = float(env.action_lim()[1][0])
    if algo == "dec_share_cbf":
        u = solve_dec_share(dec_share_data(p, ur, alpha), u_lim)[0]
    else:
        u = solve_central(central_data(p, ur, alpha), u_lim)[0].reshape(env.num_agents, -1)
    return torch.tensor(u, dtype=g.agent.dtype)


def get_cbf(env: OracleEnv, g: Graph, algo: str):
    """DecShareCBF.get_cbf -> (h, isobs); CentralizedCBF.get_cbf -> h."""
    idx, isobs = k_nearest(env, g.agent, hit_states(env, g))
    h = pairwise_h(env, g.agent, hit_states(env, g), idx)
    return (h, isobs) if algo == "dec_share_cbf" else h


def rollout_controller(env: OracleEnv, controller: Callable[[Graph], torch.Tensor], agent0, goal0, obstacles,
                       T: Optional[int] = None, enable_stop: bool = True):
    """oracle.algo.rollout with the action from `controller(graph)` (no sparsify: the baselines read the LiDAR hits
    and agent states, not the edges).  enable_stop=False steps DubinsCar without its stop mask (what DecShareCBF
    sets, dubins_car.py:138-142)."""
    T = T or env.max_episode_steps
    g = env.get_graph(agent0, goal0, obstacles)
    if not enable_stop:
        env.stop_mask = lambda agent, goal: torch.zeros(agent.shape[0], dtype=torch.bool)
    try:
        states, actions, rewards, costs, collide, finish = [], [], [], [], [], []
        with torch.no_grad():
            for _ in range(T):
                a = controller(g)
                states.append(g.agent)
                collide.append(env.collision_mask(g))
                finish.append(env.finish_mask(g))
                g, r, c = env.step(g, a)
                actions.append(a)
                rewards.append(r)
                costs.append(c)
            states.append(g.agent)
            collide.append(env.collision_mask(g))
            finish.append(env.finish_mask(g))
    finally:
        if not enable_stop:
            del env.stop_mask
    return {"states": torch.stack(states), "actions": torch.stack(actions), "rewards": torch.stack(rewards),
            "costs": torch.stack(costs), "collision": torch.stack(collide), "finish": torch.stack(finish)}
