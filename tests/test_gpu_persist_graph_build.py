"""The persistent rollout kernel's graph build against the 5-launch path (GCBF_PERSISTENT=0's graph_build_kernel), bit for
bit, on scenes built for the code that only the persistent kernel runs: the row fill of FILL_NA = 2 rows per warp
(slots s0 + 16 a of a CTA) after the LiDAR, and the cost's collision term taken from the neighbour scan's flags
(`s_col`) instead of collides_prev's walk of the previous row.

  * mixed: N = 500 (8 CTAs of 63 slots: the last CTA has 59, so its warps 11..15 run partial groups), no neighbour
    within reach on a 1.0 grid, except pairs placed at 2r - 1 ulp, 2r and 2r + 1 ulp (one in a warp group, one across
    CTAs, one at the last slots of the partial groups); rectangles next to some agents of a group and not the others,
    so that groups mix all-miss and hit LiDARs; one agent inside a rectangle.
  * parallel: the same with theta = 0 rectangles, whose edges are exactly parallel to ray 16: the NaN ray reaches every
    agent through the far-obstacle skip's vote.
  * overflow: 49 agents in a 0.1 ball on the persistent kernel's default capacity: the last row is dropped, and so is
    its collision, although it has neighbours closer than 2r.  Checked against the cost recomputed on the host from the
    kernel's own edge lists (the 5-launch path, with its batch-wide capacity, drops no row there)."""
import numpy as np
import pytest
import torch

from helpers import product_algo, product_env, product_obstacles
from test_gpu_geometry_edges import _dist, _place_pair, _sq, _states, _thresholds

F = np.float32
ENV = "DoubleIntegrator"
N_MIXED = 500


def _ws_lists(eng):
    """(row_start, row_deg, edge_src) [2][...] of the persistent kernel's workspace (rp::make_ws_layout), row starts made
    absolute: environment e's rows start at e * cap_env."""
    E, N = eng.E, eng.env.num_agents
    cap = eng._pdesc.edge_cap // E
    A, EC = E * N, E * cap
    sizes = [("msg", EC * 128), ("logit", EC), ("ag", A * 128 + 128 * 128), ("v1", A * 256 + 128 * 256), ("z", 16 * A),
             ("terms", 8 * A), ("row_start", 2 * A), ("row_deg", 2 * A), ("edge_recv", 2 * EC), ("edge_src", 2 * EC)]
    off, o = {}, 0
    for name, n in sizes:
        off[name] = o
        o += (n + 63) & ~63
    ws = eng._pws.view(torch.int32)
    rs = ws[off["row_start"]:off["row_start"] + 2 * A].view(2, A).clone()
    rd = ws[off["row_deg"]:off["row_deg"] + 2 * A].view(2, A).clone()
    es = ws[off["edge_src"]:off["edge_src"] + 2 * EC].view(2, EC).clone()
    rs += (torch.arange(A, device=rs.device) // N * cap).to(torch.int32)
    return rs.cpu().numpy(), rd.cpu().numpy(), es.cpu().numpy()


def _chain_lists(eng):
    ch = eng.chains[0]
    return ch.row_start.cpu().numpy(), ch.row_deg.cpu().numpy(), ch.edge_src.cpu().numpy()


def _rows(lists, half):
    rs, rd, es = lists
    return [es[half, rs[half, a]:rs[half, a] + rd[half, a]].tolist() for a in range(rs.shape[1])]


def _engine(scene, persistent, T, edge_cap_per_agent=None):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    agent, goal, obs = scene
    n_obs = 0 if obs is None else obs["center"].shape[1]
    env = product_env(ENV, agent.shape[1], 32.0, n_obs)
    if edge_cap_per_agent is not None:
        env.edge_cap_per_agent = edge_cap_per_agent
    algo = product_algo(env, ENV)
    eng = RolloutEngine(env, 1, T=T, n_obs=n_obs, persistent=persistent, use_cuda_graph=False)
    assert eng.persistent == persistent
    eng.set_params(algo.actor_params)
    eng.set_initial(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(),
                    product_obstacles(ENV, obs) if obs is not None else None)
    eng.run(check=False)
    torch.cuda.synchronize()
    return eng


def _record(eng):
    out = {k: getattr(eng, k).clone() for k in ("agent", "hits", "actions", "rewards", "costs")}
    out["n_edges"] = eng.counters[:, 0].clone()
    return out


# ------------------------------------------------------------------------------------------------ scenes
def _slot_agent(cta, slot, apc=63):
    return cta * apc + slot


# (i, j, measure, which): the pair's squared distance acc (the scan's value) or distance sqrtf(acc) is the largest below,
# equal to or the smallest above its threshold (two_r_sq_thr, 2r) -- one ulp from it where fp32 positions allow
PAIRS = [(5, 21, "sq", "below"), (70, 300, "sq", "at"), (_slot_agent(7, 43), _slot_agent(7, 58), "dist", "above"),
         (_slot_agent(7, 47), 130, "dist", "below"), (2, 18, "dist", "at"), (34, 400, "sq", "above")]
HIT_AGENTS = [16, 1, 49, _slot_agent(3, 7), _slot_agent(3, 55), _slot_agent(7, 31), _slot_agent(7, 58) - 2]
INSIDE_AGENT = 100


def mixed_scene(theta=0.3):
    """(agent, goal, obstacles, claims): claims are (i, j, which, distance) of the 2r pairs."""
    from gcbfplus_b200 import _lib
    two_r = _thresholds(ENV)["two_r"]
    thr = {"sq": F(_lib.sqrt_threshold(float(two_r))), "dist": two_r}
    value = {"sq": _sq, "dist": _dist}
    k = np.arange(N_MIXED)
    pos = np.stack([3.0 + 1.0 * (k % 23), 1.0 + 1.0 * (k // 23)], -1).astype(F)
    claims = []
    for n, (i, j, measure, which) in enumerate(PAIRS):
        # pairs near the origin (fine fp32 steps: exact placements exist), 0.75 apart from each other, 2 from the grid
        base = np.array([0.25 + 0.0625 * n, 0.5 + 0.75 * n], F)
        p, q = _place_pair(base, [1.0, 0.3 * n], float(two_r), [0, 1], value[measure], thr[measure], which)
        pos[i], pos[j] = p, q
        claims.append((i, j, which, value[measure](p, q), thr[measure]))
    rects = [(pos[a, 0] + 0.3, pos[a, 1] + 0.05, 0.2, 0.15, theta) for a in HIT_AGENTS]
    rects.append((pos[INSIDE_AGENT, 0], pos[INSIDE_AGENT, 1], 0.3, 0.2, theta))
    obs = dict(center=np.array([[r[:2] for r in rects]], F), width=np.array([[r[2] for r in rects]], F),
               height=np.array([[r[3] for r in rects]], F), theta=np.array([[r[4] for r in rects]], F))
    agent, goal = _states(ENV, pos, pos + F(0.3))
    return (agent, goal, obs), claims


def ball_scene(N=49, seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    r = 0.1 * np.sqrt(rng.uniform(0, 1, N))
    t = rng.uniform(0, 2 * np.pi, N)
    pos = np.stack([8.0 + r * np.cos(t), 8.0 + r * np.sin(t)], -1).astype(F)
    agent, goal = _states(ENV, pos, rng.uniform(0.5, 15.5, size=(N, 2)).astype(F))
    return agent, goal, None


def test_mixed_scene_pairs_sit_on_2r():
    _, claims = mixed_scene()
    for i, j, which, v, thr in claims:
        rel = {"below": v < thr, "at": v == thr, "above": v > thr}[which]
        assert rel, (i, j, which, v, thr)
        ulps = abs(int(np.array(v, F).view(np.int32)) - int(np.array(thr, F).view(np.int32)))
        assert ulps <= 4, (i, j, which, v, thr)


def test_overflow_scene_drops_a_colliding_row():
    agent, _, _ = ball_scene()
    p = agent[0, :, :2]
    d = np.sqrt(_sq(p[:, None], p[None]))
    np.fill_diagonal(d, np.inf)
    assert (d[-1] < _thresholds(ENV)["two_r"]).any()      # the last agent (the row that overflows) collides


# ------------------------------------------------------------------------------------------------ GPU
def _assert_same_bits(a, b):
    for k in a:
        x, y = a[k], b[k]
        same = torch.equal(x, y) or bool(((x == y) | (torch.isnan(x.float()) & torch.isnan(y.float()))).all())
        assert same, (k, float((x.float() - y.float()).abs().nan_to_num().max()))


@pytest.mark.gpu
@pytest.mark.parametrize("theta", [0.3, 0.0], ids=["mixed", "parallel"])
def test_persistent_graph_build_matches_5_launch(theta):
    scene, _ = mixed_scene(theta)
    T = 3
    eng_p = _engine(scene, True, T)
    eng_5 = _engine(scene, False, T)
    eng_p.check_overflow()
    eng_5.check_overflow()
    rec_p, rec_5 = _record(eng_p), _record(eng_5)
    _assert_same_bits(rec_p, rec_5)
    lp, l5 = _ws_lists(eng_p), _chain_lists(eng_5)
    for half in (0, 1):                      # graphs of states T - 1 and T
        assert _rows(lp, half) == _rows(l5, half), half
    hits0 = rec_p["hits"][0, 0].cpu().numpy()             # [N, R, 2] at state 0
    with np.errstate(invalid="ignore"):
        is_hit = np.linalg.norm(hits0 - scene[0][0, :, None, :2], axis=-1) <= 0.6     # misses land 1e6 rays away
    nan_ray = np.isnan(hits0).any(-1).any(-1)
    if theta == 0.0:
        assert nan_ray.all()                 # the parallel edges reach every agent
    else:
        assert not nan_ray.any()
        hit_agents = set(np.nonzero(is_hit.any(-1))[0].tolist())
        assert set(HIT_AGENTS) <= hit_agents and len(hit_agents) < 20   # groups mix hit and all-miss agents
        assert (np.abs(hits0[INSIDE_AGENT] - scene[0][0, INSIDE_AGENT, None, :2]).sum(-1) == 0).all()
    assert float(rec_p["costs"][0, 0]) > 0


@pytest.mark.gpu
def test_overflowed_row_drops_its_collision():
    T = 3
    eng = _engine(ball_scene(), True, T, edge_cap_per_agent=16)    # 48 rows per agent: 49 x 49 does not fit
    assert int(eng.counters[:, 1].max()) == 1            # some row overflowed
    rs, rd, es = _ws_lists(eng)
    half = (T - 1) % 2                                    # graph of state T - 1: the cost of step T - 1
    x = eng.agent[T - 1, 0, :, :2].cpu().numpy()
    N = x.shape[0]
    two_r = _thresholds(ENV)["two_r"]
    dropped, n_col = 0, 0
    for a in range(N):
        if rd[half, a] == 0:
            dropped += 1
            continue
        snd = [s for s in es[half, rs[half, a] + 1:rs[half, a] + rd[half, a]] if s >= 0]
        n_col += int(any(two_r > _dist(x[a], x[s]) for s in snd))
    assert dropped >= 1
    dd = np.sqrt(_sq(x[:, None], x[None]))
    np.fill_diagonal(dd, np.inf)
    assert any((dd[a] < two_r).any() for a in range(N) if rd[half, a] == 0)   # a dropped row hid a collision
    want = F(n_col) / F(N) + F(0) / F(N)
    assert float(eng.costs[T - 1, 0]) == float(want)
