"""Boundary and degenerate scenes for the graph build, the LiDAR, the k-nearest picks of the CBF-QP baselines and the
persistent rollout's edge capacity.

Random scenes almost never put a distance exactly on a threshold, a ray exactly parallel to an edge, two equal sort keys
or an edge list exactly at its capacity, so the code that exists only for those inputs is checked here with scenes built
on purpose.  Every scene is built on the host in fp32 with the oracle's own arithmetic:
  * pairs of agents whose squared distance is exactly comm_sq_thr (and the nearest achievable value below it), along x,
    y, a diagonal and z, with one agent of a pair in a full 32-candidate word of the neighbour scan and one in the tail
    word (N = 64 + 6);
  * agents whose closest LiDAR return is exactly at lidar_sq_thr, or just inside it;
  * pairs exactly at, just below and just above the 2r / unsafe / safe radii, agents exactly at an obstacle's mask radius;
  * theta = 0 rectangles: ray 16 of 32 is then exactly parallel to two edges (and rays 0, 8 and 24 too once the agent's
    coordinates round their tiny cross component away), which gives NaN in the reference whether or not the rectangle is
    in reach (the far-obstacle skip keeps that only through its `degenerate` vote);
  * an agent inside a rectangle (equal keys, then the NaN rays), on a face, next to two abutting rectangles and next
    to a duplicated one; symmetric placements with equal distances to agents and hits; coincident agents; an agent
    exactly at its goal (u_ref is NaN there, a reference quirk that must stay confined to that agent);
  * 3-D: inside a sphere (514 equal alphas), exactly 32 and exactly 33 returns (the fast / general top-k switch), a
    sphere out of reach, agents exactly at radius + r.
The CPU tests prove that every scene sits where it claims, so that a scene drifting off its boundary fails here and
does not pass silently on the GPU.  The GPU tests compare the kernels with the oracle (oracle/, tests/cbfqp_oracle.py)
and the persistent rollout with the 5-launch path on these scenes."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import cbfqp_oracle as cq
from helpers import (edge_sets_oracle, edge_sets_product, oracle_env, oracle_obstacles, oracle_params, product_algo,
                     product_env, product_obstacles)

F = np.float32
AREA = 16.0
ENVS_2D = ["SingleIntegrator", "DoubleIntegrator", "DubinsCar"]
SD = {"SingleIntegrator": 2, "DoubleIntegrator": 4, "DubinsCar": 4, "LinearDrone": 6}


# ------------------------------------------------------------------------------------------------ fp32 arithmetic
def _ulps(x, w):
    """The 2w + 1 fp32 values around x > 0, one ulp apart."""
    b = np.array(F(x)).view(np.int32)
    return (b + np.arange(-w, w + 1, dtype=np.int32)).view(F)


def _sq(p, q):
    """Squared distance in the kernels' and the oracle's order: (p - q)_0^2 + (p - q)_1^2 + ..., one rounding each."""
    d = (np.asarray(p, F) - np.asarray(q, F)).astype(F)
    acc = (d[..., 0] * d[..., 0]).astype(F)
    for c in range(1, d.shape[-1]):
        acc = (acc + d[..., c] * d[..., c]).astype(F)
    return acc


def _dist(p, q):
    return np.sqrt(_sq(p, q))           # NumPy's fp32 sqrt is correctly rounded, like sqrtf and the oracle's


def _thresholds(env_id):
    """The descriptor's fp32 thresholds (what the kernels compare against)."""
    from gcbfplus_b200.env import make_env
    d = make_env(env_id, 2, area_size=AREA, num_obs=0, device="cpu").desc(1, 0, edge_cap=64)
    return {k: F(getattr(d, k)) for k in ("comm_sq_thr", "lidar_sq_thr", "two_r", "unsafe_agent", "safe_agent",
                                          "radius", "unsafe_obs", "safe_obs")}


def _straddle(p, q0, axes, value, thr, w=64):
    """Move q0 by up to w ulps along `axes`: (q with the largest value < thr, q with value == thr or None,
    q with the smallest value > thr)."""
    grids = np.meshgrid(*[_ulps(q0[a], w) for a in axes], indexing="ij")
    q = np.tile(np.asarray(q0, F), (grids[0].size, 1))
    for a, g in zip(axes, grids):
        q[:, a] = g.reshape(-1)
    v = value(None if p is None else np.asarray(p, F)[None], q)
    lo, hi, eq = np.nonzero(v < thr)[0], np.nonzero(v > thr)[0], np.nonzero(v == thr)[0]
    return q[lo[np.argmax(v[lo])]], (q[eq[0]] if eq.size else None), q[hi[np.argmin(v[hi])]]


def _place_pair(p, direction, length, axes, value, thr, which):
    """Partner of an agent at p (shifted by steps of 1/256 until `thr` is reached exactly): the partner sits
    `length` away along `direction`, with value(p, partner) below / at / above thr.  Returns (p, partner)."""
    direction = np.asarray(direction, np.float64)
    direction /= np.linalg.norm(direction)
    for k in range(16):
        pp = (np.asarray(p, np.float64) + k / 256.0).astype(F)
        q0 = (pp + direction * length).astype(F)
        below, at, above = _straddle(pp, q0, axes, value, thr)
        if at is not None or which != "at":
            return pp, {"below": below, "at": at, "above": above}[which]
    raise AssertionError(f"no fp32 placement reaches {thr!r} exactly near {p}")


# ------------------------------------------------------------------------------------------------ scenes
class Scene:
    """agent / goal [G, N, sd]; obs: helpers' obstacle dict ([G, O, ...]) or None; claims: (name, got, relation, thr)
    tuples checked on the CPU; ties: (graph, agent, expected k-nearest idx) of the k-nearest tie placements."""

    def __init__(self, env_id, agent, goal, obs, claims, ties=(), n_rays=None):
        self.env_id, self.agent, self.goal, self.obs = env_id, agent, goal, obs
        self.claims, self.ties, self.n_rays = list(claims), list(ties), n_rays
        self.N, self.G = agent.shape[1], agent.shape[0]
        self.n_obs = 0 if obs is None else obs["center"].shape[1]


def _states(env_id, pos, goal_pos):
    """[1, N, sd] agent / goal states at rest; goal heading for DubinsCar (env/utils style: toward the goal)."""
    N, pd = pos.shape
    sd = SD[env_id]
    agent = np.zeros((1, N, sd), F)
    goal = np.zeros((1, N, sd), F)
    agent[0, :, :pd], goal[0, :, :pd] = pos, goal_pos
    if env_id == "DubinsCar":
        goal[0, :, 2] = np.arctan2(goal_pos[:, 1] - pos[:, 1], goal_pos[:, 0] - pos[:, 0])
    return agent, goal


def _grid(n, pd, spacing, origin=1.25):
    k = np.arange(n)
    cols = 8
    pos = np.zeros((n, pd), F)
    pos[:, 0] = origin + spacing * (k % cols)
    pos[:, 1] = origin + spacing * ((k // cols) % cols)
    if pd == 3:
        pos[:, 2] = origin + spacing * (k // (cols * cols))
    return pos


def pair_scene(env_id):
    """N = 70 agents, no obstacles: pairs exactly on (and next to) the neighbour, collision, unsafe and safe radii near
    the origin (small coordinates: fine fp32 steps, so exact placements exist), the other agents isolated on a 1.5
    grid further out.  Neighbour pairs at the threshold: (3, 40) scans a full word from both sides, (31, 32) sits across
    a word boundary, (10, 66) and (65, 68) reach into the tail word 64..69."""
    pd = 3 if env_id == "LinearDrone" else 2
    th = _thresholds(env_id)
    N = 70
    pos = _grid(N, pd, 1.5, origin=4.5)
    claims = []
    e = np.eye(pd)
    # off-axis direction: dx and dy move the squared distance by different amounts per ulp, so that some fp32
    # placement lands exactly on a threshold (along 45 degrees the sums collapse onto few values)
    diag = np.array([1.0, 0.6]) if pd == 2 else np.array([1.0, 0.6, 0.0])
    comm = [(31, 32, diag, "at"), (3, 40, e[0], "at"), (10, 66, e[1], "at"), (65, 68, e[0], "at"),
            (5, 45, e[0], "below"), (20, 21, e[1], "below"), (33, 60, diag, "below"), (64, 67, diag, "below")]
    if pd == 3:
        comm += [(14, 52, np.array([1.0, 0.0, 0.7]), "at"), (12, 50, e[2], "at"), (13, 51, e[2], "below")]
    used = set()
    for k, (i, j, dvec, which) in enumerate(comm):
        base = np.full(pd, 0.5, F)
        base[0], base[1] = 0.5 + 1.125 * (k % 6), 0.5 + 1.125 * (k // 6)      # dyadic: p + 0.5 is exact
        axes = [a for a in range(pd) if dvec[a] != 0]
        pos[i], pos[j] = _place_pair(base, dvec, 0.5, axes, _sq, th["comm_sq_thr"], which)
        claims.append((f"comm {which} ({i},{j})", _sq(pos[i], pos[j]), which, th["comm_sq_thr"]))
        used |= {i, j}
    free = [a for a in range(N) if a not in used]
    radii = sorted({("two_r", th["two_r"]), ("unsafe_agent", th["unsafe_agent"]), ("safe_agent", th["safe_agent"])},
                   key=lambda t: t[0])
    k = 0
    for name, r in radii:
        for which in ("below", "at", "above"):
            i, j = free.pop(0), free.pop(0)
            base = np.full(pd, 0.4, F)
            base[0], base[1] = 0.3 + 0.55 * (k // 5), 3.0 + 0.55 * (k % 5)
            k += 1
            pos[i], pos[j] = _place_pair(base, diag, float(r), [0, 1], _dist, r, which)
            claims.append((f"{name} {which} ({i},{j})", _dist(pos[i], pos[j]), which, r))
    goal = pos + F(0.2)
    agent, goal = _states(env_id, pos, goal)
    return Scene(env_id, agent, goal, None, claims)


def _rect_obs(rects):
    c = np.array([[r[0], r[1]] for r in rects], F)[None]
    return dict(center=c, width=np.array([[r[2] for r in rects]], F), height=np.array([[r[3] for r in rects]], F),
                theta=np.array([[r[4] for r in rects]], F))


def _packed_rects(rects):
    from gcbfplus_b200.env.obstacle import Rectangle
    o = _rect_obs(rects)
    return Rectangle.create(o["center"], o["width"], o["height"], o["theta"], device="cpu").packed.numpy()


def _min_hit_sq(starts, packed, n_rays=32):
    """Smallest squared distance to a non-NaN LiDAR return of each start point (oracle LiDAR, 2-D)."""
    from oracle.geometry import get_lidar, ray_table_2d
    hits = get_lidar(torch.from_numpy(np.asarray(starts, F)), oracle_obstacles(packed), ray_table_2d(n_rays, 0.5),
                     n_rays).numpy()
    acc = _sq(np.asarray(starts, F)[:, None, :], hits)
    return np.nanmin(np.where(np.isnan(acc), np.inf, acc), axis=1)


def obstacle_scene(env_id, n_rays=None):
    """2-D, 32 rectangles (the persistent kernel's limit), one agent per 2.0 cell (cells are out of each other's
    LiDAR and neighbour reach).  Every theta = 0 rectangle makes ray 16 NaN for every agent of the graph."""
    th = _thresholds(env_id)
    # structural cells 2.0 apart from x = 3.5; the exact placements sit in the column x < 1.5 (small coordinates: fine
    # fp32 steps, so positions exactly on a threshold exist)
    cell = lambda k: np.array([3.5 + 2.0 * (k % 5), 1.5 + 2.0 * (k // 5)], np.float64)
    rects, agents, claims = [], [], []
    # 0: only out-of-reach obstacles (the NaN of ray 16 comes from the far-skip's degenerate vote alone)
    c = cell(0)
    rects.append((c[0], c[1] - 1.0, 0.4, 0.4, 0.0))
    agents.append(c + [0.0, 0.2])
    # 1: a rotated rectangle in reach and theta = 0 ones out of reach (near and far in one warp)
    c = cell(1)
    rects.append((c[0] + 0.35, c[1], 0.3, 0.5, 0.7))
    agents.append(c)
    # 2: inside a theta = 0 rectangle: every ray at alpha = 0 except the NaN ones
    c = cell(2)
    rects.append((c[0], c[1], 0.5, 0.5, 0.0))
    agents.append(c + [0.05, -0.03])
    # 3: exactly on the left face (rel_xx == 0; dyadic centre and half width)
    c = np.floor(cell(3))
    rects.append((c[0], c[1], 0.5, 0.5, 0.0))
    agents.append(c - [0.25, 0.0])
    # 4: two abutting rectangles (shared edge y = c + 0.125), agent on the line of the shared edge
    c = np.floor(cell(4))
    rects += [(c[0] + 0.5, c[1], 0.5, 0.25, 0.0), (c[0] + 0.5, c[1] + 0.25, 0.5, 0.25, 0.0)]
    agents.append(c + [0.0, 0.125])
    # 5: one rectangle twice (equal alpha from two obstacles)
    c = cell(5)
    rects += [(c[0] + 0.45, c[1], 0.4, 0.4, 0.3)] * 2
    agents.append(c)
    # 6, 7: closest return just inside / exactly at lidar_sq_thr, left of a theta = 0 face (rays 15 / 17 hit first)
    for cy, which in ((2.25, "below"), (0.75, "at")):
        rect = (0.75, cy, 0.5, 0.5, 0.0)
        packed = _packed_rects([rect])[0]                  # [1, 16]
        p0 = np.array([0.5 - 0.4 * np.cos(np.pi / 16), cy], F)
        xs, ys = np.meshgrid(_ulps(p0[0], 64), _ulps(p0[1], 8), indexing="ij")
        starts = np.stack([xs.reshape(-1), ys.reshape(-1)], -1)
        m = _min_hit_sq(starts, packed)
        thr = th["lidar_sq_thr"]
        lo, eq = np.nonzero(m < thr)[0], np.nonzero(m == thr)[0]
        assert eq.size or which == "below", "no agent position puts a LiDAR return exactly at lidar_sq_thr"
        rects.append(rect)
        agents.append(starts[eq[0]] if which == "at" else starts[lo[np.argmax(m[lo])]])
    # mask radii of the obstacles: rel_xx exactly at r right of a rotated rectangle, just below r left of it
    for k, r in enumerate(sorted({float(th[n]) for n in ("radius", "unsafe_obs", "safe_obs")})):
        r = F(r)
        c = np.array([0.75, 3.75 + 1.5 * k])
        # a thin rectangle (w/2 = 2^-7): w/2 + r is then in r's binade or the next one up, so w/2 + r - w/2 can be r exactly
        rect = (c[0], c[1], 2.0 ** -6, 0.3, 0.4)
        packed = _packed_rects([rect])[0, 0]
        cs, sn = packed[4], packed[5]

        def rel_xx(p, q, packed=packed, cs=cs, sn=sn):
            rx, ry = (q[:, 0] - packed[0]).astype(F), (q[:, 1] - packed[1]).astype(F)
            return (np.abs((rx * cs + ry * sn).astype(F)) - packed[2]).astype(F)

        normal = np.array([np.cos(0.4), np.sin(0.4)])
        _, at, _ = _straddle(None, (c + (2.0 ** -7 + float(r)) * normal).astype(F), [0, 1], rel_xx, r)
        below, _, _ = _straddle(None, (c - (2.0 ** -7 + float(r)) * normal).astype(F), [0, 1], rel_xx, r)
        assert at is not None, f"no position exactly {r} from a face"
        rects.append(rect)
        agents += [below, at]
        claims.append((f"obstacle radius {r} below", rel_xx(None, below[None])[0], "below", r))
        claims.append((f"obstacle radius {r} at", rel_xx(None, at[None])[0], "at", r))
    n_agents = len(agents)
    # pad to 32 obstacles with rotated rectangles in an empty corner
    rng = np.random.Generator(np.random.PCG64(7))
    while len(rects) < 32:
        rects.append((rng.uniform(13.0, 15.5), rng.uniform(13.0, 15.5), rng.uniform(0.1, 0.4), rng.uniform(0.1, 0.4),
                      rng.uniform(0.1, 1.4)))
    pos = np.array(agents, F)
    agent, goal = _states(env_id, pos, pos + F(0.25))
    obs = _rect_obs(rects)
    packed = _packed_rects(rects)
    if n_rays in (None, 32):
        from oracle.geometry import get_lidar, ray_table_2d
        hits = get_lidar(torch.from_numpy(pos), oracle_obstacles(packed[0]), ray_table_2d(32, 0.5), 32).numpy()
        claims.append(("every agent's last hit is NaN (ray 16)", float(np.isnan(hits[:, -1]).all()), "at", 1.0))
        claims.append(("agent 0: no return in reach", float((_sq(pos[0], hits[0]) < 1).sum()), "at", 0.0))
        claims.append(("inside: every return not NaN is at the agent (alpha = 0)",
                       float((hits[2] == pos[2]).all(-1).sum() + np.isnan(hits[2]).any(-1).sum()), "at", 32.0))
        m = _min_hit_sq(pos[6:8], packed[0])
        claims.append(("lidar below", m[0], "below", th["lidar_sq_thr"]))
        claims.append(("lidar at", m[1], "at", th["lidar_sq_thr"]))
    return Scene(env_id, agent, goal, obs, claims, n_rays=n_rays)


def tie_scene(env_id):
    """Equal distances: agent 0 between agents 1 and 2 (dyadic offsets: exactly equal), agent 5 exactly on agent 4's
    closest LiDAR return, agents 6, 7, 8 coincident, agent 9 exactly at its goal."""
    from oracle.geometry import get_lidar, ray_table_2d
    rects = [(4.5, 1.5, 0.5, 0.5, 0.0), (7.0, 7.0, 0.4, 0.3, 0.0)]
    packed = _packed_rects(rects)
    pos = np.zeros((10, 2), F)
    pos[0], pos[1], pos[2], pos[3] = (1.5, 1.5), (1.625, 1.5), (1.375, 1.5), (1.5, 1.75)
    pos[4] = (4.0, 1.5)
    h4 = get_lidar(torch.from_numpy(pos[4:5]), oracle_obstacles(packed[0]), ray_table_2d(32, 0.5), 32).numpy()[0]
    pos[5] = h4[0]                                   # agent 4's closest return
    pos[6] = pos[7] = pos[8] = (1.5, 4.0)
    pos[9] = (4.0, 4.0)
    goal = pos + F(0.3)
    goal[9] = pos[9]
    agent, goal_s = _states(env_id, pos, goal)
    if env_id == "DubinsCar":
        goal_s[0, 9] = agent[0, 9]
    claims = [("0-1 / 0-2 tie", _sq(pos[0], pos[1]), "at", _sq(pos[0], pos[2])),
              ("4-5 / 4-hit0 tie", _sq(pos[4], pos[5]), "at", _sq(pos[4], h4[0])),
              ("coincident", _sq(pos[6], pos[7]), "at", F(0.0))]
    # k-nearest (stable: ties -> lower index): agent 5 (index 5) ahead of the hit (index N + 0) at the same distance
    ties = [(0, 0, [1, 2, 3]), (0, 6, [7, 8]), (0, 7, [6, 8]), (0, 4, [5, 10])]
    return Scene(env_id, agent, goal_s, _rect_obs(rects), claims, ties)


def _radius_for_returns(p, c, tab, count):
    """fp32 sphere radius giving exactly `count` rays whose line meets the sphere, or None.  Per-ray thresholds by
    bisection over fp32 bit patterns (delta grows monotonically with the radius)."""
    lo = np.zeros(tab.shape[0], np.int64)
    hi = np.full(tab.shape[0], int(np.array(F(2.0)).view(np.int32)), np.int64)
    for _ in range(32):
        mid = (lo + hi) // 2
        ok = _sphere_rows(p, c, mid.astype(np.int32).view(F), tab)
        hi = np.where(ok, mid, hi)
        lo = np.where(ok, lo, mid)
    t = np.sort(hi.astype(np.int32).view(F))
    return t[count - 1] if t[count - 1] < t[count] else None


def _sphere_rows(p, c, rho, tab):
    """Does the line of ray r meet the sphere of radius rho[r] (delta >= 0)?  The oracle's operation order."""
    x1 = np.asarray(p, F)
    x2 = (x1[None] + tab).astype(F)
    d = (x2 - x1[None]).astype(F)
    rmax = np.sqrt(_sq(x2, x1[None]))
    A = (rmax * rmax).astype(F)
    e = (x1 - np.asarray(c, F)).astype(F)
    B = (F(2) * ((d[:, 0] * e[0] + d[:, 1] * e[1]).astype(F) + d[:, 2] * e[2]).astype(F)).astype(F)
    C = (((e[0] * e[0] + e[1] * e[1]).astype(F) + e[2] * e[2]).astype(F) - (rho * rho).astype(F)).astype(F)
    delta = ((B * B).astype(F) - ((F(4) * A).astype(F) * C).astype(F)).astype(F)
    return delta >= 0


def _lidar3d(pos, centers, radii, R):
    from oracle.geometry import Sphere, get_lidar, ray_table_3d
    sph = Sphere(torch.from_numpy(np.asarray(centers, F)), torch.from_numpy(np.asarray(radii, F)))
    return get_lidar(torch.from_numpy(np.asarray(pos, F)), sph, ray_table_3d(32, 0.5), R).numpy()


def _n_returns(p, center, rho):
    from oracle.geometry import Sphere, ray_table_3d
    tab = ray_table_3d(32, 0.5)
    st = torch.from_numpy(np.asarray(p, F))[None].expand(tab.shape[0], 3)
    a = Sphere(torch.from_numpy(np.asarray([center], F)), torch.from_numpy(np.asarray([rho], F))).raytracing(st, st + tab)
    return int((a[:, 0] < 1e6).sum())


def sphere_scene():
    """LinearDrone, 4 graphs of 4 agents and one sphere each: g0 agent 0 sees exactly 32 returns (fast path), g1
    exactly 33 (general path); g2 agent 0 inside the sphere (514 alphas of 0), agents 1-3 exactly at radius, radius + r
    and radius + 1.5 r from its centre; g3 a sphere beyond the rays' reach (returns at alpha = 1 behind and ahead)."""
    from oracle.geometry import ray_table_3d
    th = _thresholds("LinearDrone")
    tab = ray_table_3d(32, 0.5).numpy()
    G, N = 4, 4
    pos = np.zeros((G, N, 3), F)
    centers = np.zeros((G, 1, 3), F)
    radii = np.zeros((G, 1), F)
    far = np.array([[0.0, 0.0, 0.0], [2.5, 0.3, 0.2], [0.4, 2.6, 0.1], [0.2, 0.5, 2.7]])
    claims = []
    u = np.array([0.6, 0.48, 0.64])
    for g, count in ((0, 32), (1, 33)):
        rho = None
        for k in range(32):
            p = np.array([1.0, 1.0, 1.0], F)
            c = (p + (0.3 + 0.01 * k) * u).astype(F)
            rho = _radius_for_returns(p, c, tab, count)
            if rho is not None:
                break
        assert rho is not None, f"no sphere radius gives exactly {count} returns"
        pos[g] = (p + far).astype(F)
        centers[g, 0], radii[g, 0] = c, rho
        claims.append((f"g{g}: {count} returns", float(_n_returns(pos[g, 0], c, rho)), "at", float(count)))
    # g2: inside, and exactly on the inside / mask boundaries (sqrt(d^2) == radius + r, `<=`)
    c2 = np.array([1.0, 1.0, 1.0], F)
    rho2 = F(0.15)
    pos[2, 0] = c2
    for a, r, dvec, axes in ((1, F(0.0), (1.0, 0.0, 0.3), [0, 2]), (2, th["radius"], (0.0, -1.0, 0.3), [1, 2]),
                             (3, th["unsafe_obs"], (0.3, 0.0, 1.0), [0, 2])):
        tgt = F(rho2 + r)
        dvec = np.array(dvec) / np.linalg.norm(dvec)
        _, q, _ = _straddle(c2, (c2 + dvec * float(tgt)).astype(F), axes, _dist, tgt)
        assert q is not None, f"no position exactly radius + {float(r)} from the centre"
        pos[2, a] = q
        claims.append((f"g2 agent {a} at radius + {float(r)}", _dist(c2, q), "at", tgt))
    centers[2, 0], radii[2, 0] = c2, rho2
    claims.append(("g2 agent 0 at the centre", float(_n_returns(pos[2, 0], c2, rho2)), "at", 514.0))
    # g3: sphere 0.8 away (beyond the 0.5 rays): every ray whose line meets it returns alpha = 1
    pos[3] = (np.array([1.0, 1.0, 1.0]) + far).astype(F)
    centers[3, 0], radii[3, 0] = (pos[3, 0] + 0.8 * u).astype(F), F(0.2)
    n3 = _n_returns(pos[3, 0], centers[3, 0], radii[3, 0])
    claims.append(("g3 returns (fast path)", float(0 < n3 <= 32), "at", 1.0))
    goal = pos + F(0.2)
    agent = np.zeros((G, N, 6), F)
    goal_s = np.zeros((G, N, 6), F)
    agent[..., :3], goal_s[..., :3] = pos, goal
    return Scene("LinearDrone", agent, goal_s, dict(center=centers, radius=radii), claims)


SCENES = {
    "pairs": lambda env_id: pair_scene(env_id),
    # 32 rays for every env (DubinsCar defaults to 16): the LiDAR placements are made for ray 16 being horizontal
    "obstacles": lambda env_id: obstacle_scene(env_id, n_rays=32 if env_id == "DubinsCar" else None),
    "obstacles16": lambda env_id: obstacle_scene(env_id, n_rays=16),
    "ties": lambda env_id: tie_scene(env_id),
    "spheres": lambda env_id: sphere_scene(),
}
SCENE_CASES = ([("pairs", e) for e in ENVS_2D + ["LinearDrone"]] + [("obstacles", e) for e in ENVS_2D] +
               [("obstacles16", "DoubleIntegrator"), ("spheres", "LinearDrone")] + [("ties", e) for e in ENVS_2D])
_CACHE = {}


def scene(name, env_id):
    if (name, env_id) not in _CACHE:
        _CACHE[(name, env_id)] = SCENES[name](env_id)
    return _CACHE[(name, env_id)]


# ================================================================================================ CPU: the scenes
@pytest.mark.parametrize("name,env_id", SCENE_CASES)
def test_scene_sits_on_its_boundary(name, env_id):
    s = scene(name, env_id)
    assert s.claims or s.ties
    for what, got, rel, thr in s.claims:
        got, thr = F(got), F(thr)
        if rel == "at":
            assert got == thr, (what, got, thr)
        elif rel == "below":
            assert got < thr and thr - got <= F(4e-6) * max(thr, F(1e-3)), (what, got, thr)
        else:
            assert got > thr and got - thr <= F(4e-6) * max(thr, F(1e-3)), (what, got, thr)
    if s.ties:
        oenv = oracle_env(env_id, s.N, AREA, s.n_obs)
        og = oenv.get_graph(torch.from_numpy(s.agent[0]), torch.from_numpy(s.goal[0]),
                            oracle_obstacles(_packed_rects_from(s)[0]))
        idx, _ = cq.k_nearest(oenv, og.agent, cq.hit_states(oenv, og))
        for g, i, want in s.ties:
            assert idx[i, :len(want)].tolist() == want, (i, idx[i].tolist(), want)


def test_threshold_constants_match_the_oracle():
    """The descriptor's radii are the oracle's fp32 constants, so a scene on a descriptor threshold is on the oracle's."""
    for env_id in ENVS_2D + ["LinearDrone"]:
        th = _thresholds(env_id)
        oenv = oracle_env(env_id, 2, AREA, 0)
        r = oenv.r
        assert th["two_r"] == F(oenv._c(r * 2).item())
        assert np.sqrt(th["comm_sq_thr"]) >= F(0.5) > np.sqrt(np.nextafter(th["comm_sq_thr"], F(0)))
        assert np.sqrt(th["lidar_sq_thr"]) >= F(0.5 - 1e-1) > np.sqrt(np.nextafter(th["lidar_sq_thr"], F(0)))


def _packed_rects_from(s):
    from gcbfplus_b200.env.obstacle import Rectangle, Sphere
    if s.obs is None:
        return np.zeros((s.G, 0, 16), F)
    if "radius" in s.obs:
        return Sphere.create(s.obs["center"], s.obs["radius"], device="cpu").packed.numpy()
    return Rectangle.create(s.obs["center"], s.obs["width"], s.obs["height"], s.obs["theta"], device="cpu").packed.numpy()


# ================================================================================================ GPU
def _product_graph(s, edge_cap_per_agent=128):
    env = product_env(s.env_id, s.N, AREA, s.n_obs, s.n_rays)
    env.edge_cap_per_agent = edge_cap_per_agent
    pobs = product_obstacles(s.env_id, s.obs) if s.obs is not None else None
    graph = env.get_graph(torch.from_numpy(s.agent).cuda(), torch.from_numpy(s.goal).cuda(), pobs)
    torch.cuda.synchronize()
    graph.check_overflow()
    return env, graph, pobs


def _oracle_graphs(s, env):
    oenv = oracle_env(s.env_id, s.N, AREA, s.n_obs, s.n_rays)
    packed = _packed_rects_from(s)
    out = []
    for g in range(s.G):
        oobs = oracle_obstacles(packed[g]) if s.n_obs > 0 else None
        dense = oenv.get_graph(torch.from_numpy(s.agent[g]), torch.from_numpy(s.goal[g]), oobs)
        out.append((dense, oenv.sparsify(dense)))
    return oenv, out


@pytest.mark.gpu
@pytest.mark.parametrize("name,env_id", SCENE_CASES)
def test_graph_build_and_masks_on_boundaries(name, env_id):
    """(a) hits bit-exact (NaN == NaN), edge sets, edge count and the four masks equal to the oracle's."""
    s = scene(name, env_id)
    env, graph, _ = _product_graph(s)
    oenv, ogs = _oracle_graphs(s, env)
    hits = graph.hits.cpu().numpy()
    masks = {k: getattr(env, k + "_mask")(graph).cpu().numpy() for k in ("unsafe", "collision", "finish", "safe")}
    n_edges = 0
    for g, (dense, og) in enumerate(ogs):
        ohits = dense.states[2 * s.N:-1, :env.pos_dim].reshape(s.N, env.n_hits, env.pos_dim).numpy()
        np.testing.assert_array_equal(hits[g], ohits)
        assert edge_sets_product(graph, g, s.N) == edge_sets_oracle(og, s.N, env.n_hits)
        for k, v in masks.items():
            np.testing.assert_array_equal(v[g], getattr(oenv, k + "_mask")(dense).numpy(), err_msg=f"{k} mask")
        n_edges += og.edges.shape[0]
    assert graph.n_edge == n_edges


def _same_nan_close(got, want, atol, what):
    got, want = np.asarray(got), np.asarray(want)
    np.testing.assert_array_equal(np.isnan(got), np.isnan(want), err_msg=f"{what}: NaN pattern")
    np.testing.assert_allclose(got, want, atol=atol, rtol=0, err_msg=what)


@pytest.mark.gpu
@pytest.mark.parametrize("name,env_id", SCENE_CASES)
def test_network_and_step_on_boundaries(name, env_id, gemm_path):
    """(b) h, pi, act and env.step against the oracle at the gnn tests' tolerances; the cost exactly; NaN (u_ref at the
    goal) in exactly the oracle's entries."""
    from oracle.algo import act, get_cbf
    from oracle.nn import net_forward
    from test_gpu_gnn import TOL
    tol = TOL[gemm_path]
    s = scene(name, env_id)
    env, graph, _ = _product_graph(s)
    algo = product_algo(env, env_id)
    h = algo.get_cbf(graph).cpu().numpy()
    pi = algo.get_action(graph).cpu().numpy()
    a = algo.act(graph)
    nxt = env.step(graph, a)
    torch.cuda.synchronize()
    oenv, ogs = _oracle_graphs(s, env)
    ap, cp = oracle_params(env_id)
    with torch.no_grad():
        for g, (_, og) in enumerate(ogs):
            _same_nan_close(h[g], get_cbf(cp, og).numpy(), tol, "h")
            _same_nan_close(pi[g], net_forward(ap, og, "actor").numpy(), tol, "pi")
            _same_nan_close(a[g].cpu().numpy(), act(oenv, ap, og).numpy(), 2 * tol + 1e-5, "action")
            og2, r, c = oenv.step(og, torch.from_numpy(a[g].cpu().numpy()))
            _same_nan_close(nxt.graph.agent[g].cpu().numpy(), og2.agent.numpy(), 1e-6, "next state")
            _same_nan_close(nxt.reward[g].cpu().numpy(), r.numpy(), 1e-5 * max(1.0, abs(float(r))), "reward")
            assert nxt.cost[g].item() == c.item(), (nxt.cost[g].item(), c.item())
    if name == "ties" and env_id != "DubinsCar":
        # agent 9 sits exactly at its goal: NaN u_ref, NaN action and next state for it alone
        bad = ~torch.isfinite(a).all(-1).cpu()
        assert bad[0].nonzero().flatten().tolist() == [9]
        assert bool(torch.isfinite(nxt.graph.agent[0, :9]).all())


def _run_engine(env, s, persistent, T, E=1):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    algo = product_algo(env, s.env_id)
    pobs = product_obstacles(s.env_id, s.obs) if s.obs is not None else None
    eng = RolloutEngine(env, E, T=T, n_obs=s.n_obs, persistent=persistent)
    assert eng.persistent == persistent
    eng.set_params(algo.actor_params)
    eng.set_initial(torch.from_numpy(s.agent).cuda(), torch.from_numpy(s.goal).cuda(), pobs)
    return eng


def _record(eng):
    out = {k: getattr(eng, k).clone() for k in ("agent", "hits", "actions", "rewards", "costs")}
    out["n_edges"] = eng.counters[:, 0].clone()
    return out


def _assert_same_bits(a, b):
    for k in a:
        x, y = a[k], b[k]
        same = torch.equal(x, y) or bool(((x == y) | (torch.isnan(x.float()) & torch.isnan(y.float()))).all())
        assert same, (k, float((x.float() - y.float()).abs().nan_to_num().max()))


ROLLOUT_CASES = [("pairs", "DoubleIntegrator"), ("pairs", "SingleIntegrator"), ("obstacles", "DoubleIntegrator"),
                 ("obstacles", "SingleIntegrator"), ("obstacles16", "DoubleIntegrator"), ("ties", "DoubleIntegrator"),
                 ("ties", "SingleIntegrator"), ("ties", "DubinsCar")]


@pytest.mark.gpu
@pytest.mark.parametrize("name,env_id", ROLLOUT_CASES)
def test_rollout_paths_agree_on_boundaries(name, env_id):
    """(c) the persistent kernel (n_obs = 32, 0; 16 rays) and the 5-launch path over 3 steps: the same bits (DubinsCar:
    its 2e-4 closed-loop bar); step 0 equal to the oracle's graph."""
    s = scene(name, env_id)
    env = product_env(env_id, s.N, AREA, s.n_obs, s.n_rays)
    recs = []
    for persistent in (True, False):
        eng = _run_engine(env, s, persistent, T=3)
        eng.run()
        torch.cuda.synchronize()
        recs.append(_record(eng))
    if env_id == "DubinsCar":
        for k in recs[0]:
            if k not in ("hits", "n_edges"):
                assert float((recs[0][k].float() - recs[1][k].float()).abs().nan_to_num().max()) <= 2e-4, k
        assert torch.equal(recs[0]["n_edges"], recs[1]["n_edges"])
    else:
        _assert_same_bits(*recs)
    oenv, ogs = _oracle_graphs(s, env)
    dense, og = ogs[0]
    ohits = dense.states[2 * s.N:-1, :env.pos_dim].reshape(s.N, env.n_hits, env.pos_dim).numpy()
    np.testing.assert_array_equal(recs[0]["hits"][0, 0].cpu().numpy(), ohits)
    assert int(recs[0]["n_edges"][0]) == og.edges.shape[0]
    if name == "ties" and env_id != "DubinsCar":
        fin = torch.isfinite(recs[0]["agent"][1:, 0]).all(-1).cpu()      # [T, N]: only agent 9 (at its goal) goes NaN
        assert fin[:, :9].all() and not fin[:, 9].any()


@pytest.mark.gpu
@pytest.mark.parametrize("name,env_id", [("ties", e) for e in ENVS_2D] + [("obstacles", "DoubleIntegrator")])
def test_k_nearest_ties_and_nan_hits(name, env_id):
    """(d) DecShareCBF.pairwise index sets and isobs bit-exact against the oracle: ties to the lower index, NaN hits
    after every number."""
    from gcbfplus_b200.algo import make_algo
    s = scene(name, env_id)
    env, graph, _ = _product_graph(s)
    dec = make_algo("dec_share_cbf", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                    action_dim=env.action_dim, n_agents=env.num_agents)
    pw = dec.pairwise(graph)
    idx, isobs = pw["idx"].cpu().numpy(), pw["isobs"].cpu().numpy()
    oenv, ogs = _oracle_graphs(s, env)
    for g, (dense, _) in enumerate(ogs):
        oidx, oisobs = cq.k_nearest(oenv, dense.agent, cq.hit_states(oenv, dense))
        np.testing.assert_array_equal(idx[g], oidx.numpy())
        np.testing.assert_array_equal(isobs[g], oisobs.numpy())
        hits = graph.hits[g].cpu().numpy()
        picked_hits = idx[g][idx[g] >= s.N] - s.N
        rows = np.nonzero(idx[g] >= s.N)[0]
        assert not np.isnan(hits[rows, picked_hits]).any(), "a NaN hit was picked ahead of a number"
    for g, i, want in s.ties:
        assert idx[g, i, :len(want)].tolist() == want


# ------------------------------------------------------------------------------------------------ 3-D n_hits (C ABI)
@pytest.mark.gpu
@pytest.mark.parametrize("R", [16, 24, 32])
def test_3d_top_k_keeps_n_hits_returns(R):
    """gcbf_graph_build with a LinearDrone descriptor of n_hits = R (the header allows up to 32): argsort(alpha)[:R]
    of the 514 rays equal to the oracle's get_lidar(max_returns=R), fast path (few returns: most hit slots are the
    first missing rays in ray order) and general path alike."""
    import ctypes as C
    from gcbfplus_b200 import _lib
    s = sphere_scene()
    env = product_env("LinearDrone", s.N, AREA, 1)
    G, N = s.G, s.N
    pobs = product_obstacles("LinearDrone", s.obs)
    agent = torch.from_numpy(s.agent).cuda()
    d = env.desc(G, 1, edge_cap=G * N * (N + R))
    d.n_hits = R
    hits = torch.full((G, N, R, 3), float("nan"), device="cuda")
    i32 = dict(dtype=torch.int32, device="cuda")
    rs, rd = torch.empty(G * N, **i32), torch.empty(G * N, **i32)
    er, es, cnt = torch.zeros(d.edge_cap, **i32), torch.zeros(d.edge_cap, **i32), torch.zeros(4, **i32)
    rc = env.lib.gcbf_graph_build(C.byref(d), _lib.ptr(agent), _lib.ptr(pobs.packed), _lib.ptr(env.ray_table),
                                  _lib.ptr(hits), _lib.ptr(rs), _lib.ptr(rd), _lib.ptr(er), _lib.ptr(es), _lib.ptr(cnt), 1,
                                  env._stream())
    _lib.check(rc, "gcbf_graph_build")
    torch.cuda.synchronize()
    got = hits.cpu().numpy()
    packed = pobs.packed.cpu().numpy()
    for g in range(G):
        want = _lidar3d(s.agent[g, :, :3], packed[g, :, :3], packed[g, :, 3], R)
        np.testing.assert_array_equal(got[g], want, err_msg=f"graph {g}")
    # the same through the obstacle-free path (every ray misses: all R slots are the first R rays)
    d0 = env.desc(G, 0, edge_cap=G * N * (N + R))
    d0.n_hits = R
    rc = env.lib.gcbf_graph_build(C.byref(d0), _lib.ptr(agent), None, _lib.ptr(env.ray_table), _lib.ptr(hits),
                                  _lib.ptr(rs), _lib.ptr(rd), _lib.ptr(er), _lib.ptr(es), _lib.ptr(cnt), 1, env._stream())
    _lib.check(rc, "gcbf_graph_build")
    torch.cuda.synchronize()
    from oracle.geometry import get_lidar, ray_table_3d
    for g in range(G):
        want = get_lidar(torch.from_numpy(s.agent[g, :, :3]), None, ray_table_3d(32, 0.5), R).numpy()
        np.testing.assert_array_equal(hits[g].cpu().numpy(), want)


# ------------------------------------------------------------------------------------------------ edge capacity
def _ball(N, n_clustered, seed=0):
    """DoubleIntegrator at rest: agents 0..n_clustered-1 inside one 0.1-radius ball, the rest spread over the area."""
    rng = np.random.Generator(np.random.PCG64(seed))
    pos = np.zeros((N, 2), F)
    r = 0.1 * np.sqrt(rng.uniform(0, 1, n_clustered))
    t = rng.uniform(0, 2 * np.pi, n_clustered)
    pos[:n_clustered] = np.stack([8.0 + r * np.cos(t), 8.0 + r * np.sin(t)], -1)
    pos[n_clustered:] = rng.uniform(0.5, AREA - 0.5, size=(N - n_clustered, 2))
    pos[n_clustered:][np.hypot(*(pos[n_clustered:] - 8.0).T) < 1.0] += 2.0     # keep the spread agents off the ball
    agent, goal = _states("DoubleIntegrator", pos, rng.uniform(0.5, AREA - 0.5, size=(N, 2)).astype(F))
    return Scene("DoubleIntegrator", agent, goal, None, [])


def test_capacity_scenes_fill_what_they_claim():
    """N = 48 in a 0.1 ball: every agent is every other's neighbour (48 rows per agent: 48 x 48 = the persistent
    kernel's per-environment capacity at the default edge_cap_per_agent); N = 49 is one agent over."""
    for N in (48, 49):
        p = _ball(N, N).agent[0, :, :2]
        assert (_sq(p[:, None], p[None]) < F(0.25)).all()
    s = _ball(200, 50)
    p = s.agent[0, :, :2]
    assert (_sq(p[:50, None], p[None, :50]) < F(0.25)).all()


def _capacity_run(N, n_clustered, persistent, edge_cap_per_agent=16, T=3):
    s = _ball(N, n_clustered)
    env = product_env("DoubleIntegrator", N, AREA, 0)
    env.edge_cap_per_agent = edge_cap_per_agent
    eng = _run_engine(env, s, persistent, T)
    eng.run(check=False)
    torch.cuda.synchronize()
    return eng


@pytest.mark.gpu
def test_persistent_capacity_exactly_full():
    eng = _capacity_run(48, 48, persistent=True)
    assert eng._pdesc.edge_cap == 48 * 48
    eng.check_overflow()
    assert eng.counters[:, 0].tolist() == [48 * 48] * 4
    ref = _capacity_run(48, 48, persistent=False, edge_cap_per_agent=64)
    ref.check_overflow()
    _assert_same_bits(_record(eng), _record(ref))


@pytest.mark.gpu
@pytest.mark.parametrize("persistent", [True, False])
def test_capacity_one_agent_over_is_reported(persistent):
    eng = _capacity_run(49, 49, persistent=persistent)
    with pytest.raises(RuntimeError, match="overflow"):
        eng.check_overflow()


def _pair_segment_outcome():
    """Run the clustered N = 200 scene on the persistent kernel: 'OVERFLOW' or 'OK' (this or a child process)."""
    eng = _capacity_run(200, 50, persistent=True)
    try:
        eng.check_overflow()
    except RuntimeError as e:
        assert "overflow" in str(e)
        return "OVERFLOW"
    return "OK"


@pytest.mark.gpu
def test_pair_segment_overflow_is_reported():
    """Agents 0..49 in one ball: 2500 rows in the first 50 agents.  With one cluster per environment (segment = the
    environment's 9600 rows) that fits and equals the 5-launch path; in pair mode (GCBF_PERSIST_SOFT=1: a pair of CTAs
    owns cap_env / 4 = 2400 rows) the segment overflows while the environment fits, and that must be reported."""
    assert _pair_segment_outcome() == "OK"
    a = _record(_capacity_run(200, 50, persistent=True))
    b = _record(_capacity_run(200, 50, persistent=False, edge_cap_per_agent=64))
    _assert_same_bits(a, b)
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_gpu_geometry_edges as t; "
            "print('OUTCOME', t._pair_segment_outcome())" % (here, os.path.dirname(here)))
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GCBF_PERSIST_SOFT="1"), capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    assert [l for l in out.stdout.splitlines() if l.startswith("OUTCOME")][0].split()[1] == "OVERFLOW"
