"""CPU: the CBF-QP baseline oracle (tests/cbfqp_oracle.py) against closed-form answers and independent solvers."""
import numpy as np
import pytest
import torch

import cbfqp_oracle as cq
from helpers import ENVS, oracle_env
from oracle.qp import kkt_residual, solve_qp_slsqp

FAR = 1e6


def _scene(env_id, pos, vel=None, hits=None, dtype=torch.float64):
    """Agents at `pos` (+ velocity / DubinsCar heading+speed), R = len(hits[0]) hit nodes per agent."""
    env = oracle_env(env_id, len(pos), 4.0, 0, dtype=dtype)
    sd, pd = env.state_dim, env.pos_dim
    x = torch.zeros(len(pos), sd, dtype=dtype)
    x[:, :pd] = torch.tensor(pos, dtype=dtype)
    if vel is not None:
        x[:, pd:] = torch.tensor(vel, dtype=dtype)
    hits = hits if hits is not None else [[[FAR] * pd] for _ in pos]
    hs = torch.zeros(len(pos), len(hits[0]), sd, dtype=dtype)
    hs[..., :pd] = torch.tensor(hits, dtype=dtype)
    return env, x, hs


def _hand(env_id, env, x, i, j):
    """Closed-form h and dh/dx_i for agent i against agent j (float64)."""
    pd = env.pos_dim
    dp = (x[i, :pd] - x[j, :pd]).numpy()
    off = cq.h_offset(env)
    if env_id == "SingleIntegrator":
        return dp @ dp - off, 2 * dp
    if env_id == "DubinsCar":
        th, s = float(x[i, 2]), float(x[i, 3])
        vi = s * np.array([np.cos(th), np.sin(th)])
        vj = float(x[j, 3]) * np.array([np.cos(float(x[j, 2])), np.sin(float(x[j, 2]))])
        dv = vi - vj
        gi = np.concatenate([2 * dv + 10 * dp, [2 * dp @ (s * np.array([-np.sin(th), np.cos(th)])),
                                                2 * dp @ np.array([np.cos(th), np.sin(th)])]])
        return 2 * dp @ dv + 5 * (dp @ dp - off), gi
    dv = (x[i, pd:] - x[j, pd:]).numpy()
    c = cq.GAIN[env_id]
    return 2 * dp @ dv + c * (dp @ dp - off), np.concatenate([2 * dv + 2 * c * dp, 2 * dp])


@pytest.mark.parametrize("env_id", ENVS)
def test_known_answers_three_agents(env_id):
    """Three agents within distance 10 of each other, the only hit far away: each picks the two others (nearest
    first), then itself (distance 100).  h and the jacfwd Jacobian match the closed form in float64."""
    pd = 3 if env_id == "LinearDrone" else 2
    pos = [[0.0, 0.0, 0.1][:pd], [0.3, 0.1, 0.0][:pd], [-0.5, 0.4, 0.2][:pd]]
    if env_id == "DubinsCar":
        vel = [[0.4, 0.3], [-1.2, 0.5], [2.0, -0.2]]
    elif env_id == "SingleIntegrator":
        vel = None
    else:
        vel = [[0.1, -0.2, 0.3][:pd], [-0.3, 0.2, 0.0][:pd], [0.05, 0.4, -0.1][:pd]]
    env, x, hs = _scene(env_id, pos, vel)
    p = cq.pairwise(env, x, hs)
    d = lambda a, b: float(((x[a, :pd] - x[b, :pd]) ** 2).sum())
    for i in range(3):
        others = sorted([j for j in range(3) if j != i], key=lambda j: d(i, j))
        assert p["idx"][i].tolist() == others + [i]
        assert not p["isobs"][i].any()
        for k, j in enumerate(others):
            h, gi = _hand(env_id, env, x, i, j)
            assert abs(float(p["h"][i, k]) - h) <= 1e-12 * max(1.0, abs(h))
            np.testing.assert_allclose(p["hx"][i, k, i].numpy(), gi, rtol=1e-12, atol=1e-12)
            gj = p["hx"][i, k, j].numpy()
            if env_id == "DubinsCar":    # dh/dx_j through agent j's own heading / speed
                np.testing.assert_allclose(gj[:2], -gi[:2], rtol=1e-12, atol=1e-12)
            else:
                np.testing.assert_allclose(gj, -gi, rtol=1e-12, atol=1e-12)
            rest = [q for q in range(3) if q not in (i, j)]
            assert torch.all(p["hx"][i, k, rest] == 0)
        # self pick: constant distance 100, zero gradient
        c = cq.GAIN.get(env_id, 1.0)
        assert float(p["h"][i, 2]) == pytest.approx(c * (100 - cq.h_offset(env)), rel=1e-12)
        assert torch.all(p["hx"][i, 2] == 0) and torch.all(p["lg_self"][i, 2] == 0) and float(p["lf_h"][i, 2]) == 0


def test_stable_tie_breaking():
    """Equidistant candidates keep index order (stable argsort), hits after agents at equal distance."""
    env, x, hs = _scene("SingleIntegrator", [[0.0, 0.0], [1.0, 0.0], [-1.0, 0.0], [0.0, 5.0]],
                        hits=[[[0.0, 1.0], [0.0, -1.0]], [[FAR, FAR]] * 2, [[FAR, FAR]] * 2, [[FAR, FAR]] * 2])
    idx, isobs = cq.k_nearest(env, x, hs)
    assert idx[0].tolist() == [1, 2, 4]          # agents 1, 2 and hit 0 (index N + 0) all at distance 1
    assert isobs[0].tolist() == [False, False, True]
    env, x, hs = _scene("SingleIntegrator", [[0.0, 0.0], [3.0, 0.0], [0.0, -1.0]],
                        hits=[[[1.0, 0.0], [0.0, 1.0]], [[FAR, FAR]] * 2, [[FAR, FAR]] * 2])
    idx, _ = cq.k_nearest(env, x, hs)
    assert idx[0].tolist() == [2, 3, 4]          # agent 2, then the two hits at the same distance, in order


def test_responsibility_scales_b_only():
    env, x, hs = _scene("DoubleIntegrator", [[0.0, 0.0], [0.2, 0.0], [3.0, 3.0]],
                        [[0.2, 0.0], [-0.2, 0.0], [0.0, 0.0]], hits=[[[0.0, 0.15]], [[FAR, FAR]], [[FAR, FAR]]])
    p = cq.pairwise(env, x, hs)
    assert p["isobs"][0].tolist() == [True, False, False]
    ur = torch.zeros(3, 2, dtype=torch.float64)
    d = cq.dec_share_data(p, ur, alpha=1.0)
    np.testing.assert_array_equal(d["Lg"], p["lg_self"].numpy())
    full = (p["lf_h"] + p["h"]).numpy()
    np.testing.assert_array_equal(d["b"][0], full[0] * np.array([1.0, 0.5, 0.5]))


def _qp_scene(env_id, N, seed):
    """Crowded float64 scene: agents close together and closing in, hits scattered around them, so that CBF rows are
    active."""
    rng = np.random.default_rng(seed)
    env = oracle_env(env_id, N, 1.0, 0, dtype=torch.float64)
    sd, pd = env.state_dim, env.pos_dim
    x = torch.zeros(N, sd, dtype=torch.float64)
    x[:, :pd] = torch.tensor(rng.uniform(0, 0.5, (N, pd)))
    if env_id == "DubinsCar":
        x[:, 2] = torch.tensor(rng.uniform(-np.pi, np.pi, N))
        x[:, 3] = torch.tensor(rng.uniform(-0.5, 0.5, N))
    elif sd > pd:
        x[:, pd:] = torch.tensor(rng.uniform(-0.5, 0.5, (N, sd - pd)))
    goal = torch.zeros(N, sd, dtype=torch.float64)
    goal[:, :pd] = torch.tensor(rng.uniform(0, 1.0, (N, pd)))
    R = 4
    hs = torch.zeros(N, R, sd, dtype=torch.float64)
    hs[..., :pd] = x[:, None, :pd] + torch.tensor(rng.uniform(-0.15, 0.15, (N, R, pd)))
    return env, x, goal, hs


@pytest.mark.parametrize("env_id", ENVS)
def test_qps_agree_with_slsqp_and_kkt(env_id):
    env, x, goal, hs = _qp_scene(env_id, 6, seed=4)
    p = cq.pairwise(env, x, hs)
    ur = env.u_ref(x, goal)
    u_lim = float(env.action_lim()[1][0])
    # DecShareCBF: one problem per agent
    d = cq.dec_share_data(p, ur, alpha=1.0)
    u, r, lam, _ = cq.solve_dec_share(d, u_lim)
    n_active = 0
    for i in range(env.num_agents):
        us, rs, _ = solve_qp_slsqp(d["Lg"][i], d["b"][i], d["u_ref"][i], u_lim)
        np.testing.assert_allclose(u[i], us, atol=1e-6)
        np.testing.assert_allclose(r[i], rs, atol=1e-5)   # SLSQP's relaxations stop a few 1e-6 short
        kkt = kkt_residual(d["Lg"][i], d["b"][i], d["u_ref"][i], u_lim, u[i], r[i], lam[i])
        assert max(kkt.values()) <= 1e-9, kkt
        n_active += int((lam[i] > 1e-9).sum())
    assert n_active > 0, "no CBF row is active: the scene does not test the QP"
    # CentralizedCBF: one problem per graph
    d = cq.central_data(p, ur, alpha=1.0)
    u, r, lam, _ = cq.solve_central(d, u_lim)
    us, rs, _ = solve_qp_slsqp(d["Lg"], d["b"], d["u_ref"], u_lim)
    np.testing.assert_allclose(u, us, atol=1e-6)
    np.testing.assert_allclose(r, rs, atol=1e-5)
    kkt = kkt_residual(d["Lg"], d["b"], d["u_ref"], u_lim, u, r, lam)
    assert max(kkt.values()) <= 1e-9, kkt
    assert (lam > 1e-9).any(), "no CBF row is active: the scene does not test the QP"
    # the sparse form the GPU tests use on the kernel's per-row blocks is the same matrix
    sparse = cq.central_from_blocks(p["idx"].numpy(), p["lg_self"].numpy(), p["lg_other"].numpy())
    np.testing.assert_array_equal(sparse.toarray(), d["Lg"])


def test_h_offset_rounding_of_the_device_constant():
    """csrc/cbfqp.cu derives 4 (1.01 r)^2 from the descriptor's fp32 4 r^2 as fp32(1.0201 * four_r_sq); that must be
    the fp32 the reference's weak typing makes of the python float."""
    for env_id in ENVS:
        env = oracle_env(env_id, 2, 1.0, 0)
        r = env.r
        four_r_sq = np.float32(4 * r ** 2)
        want = np.float32(cq.h_offset(env))
        got = np.float32(1.0201 * float(four_r_sq)) if env_id in ("SingleIntegrator", "LinearDrone") else four_r_sq
        assert got == want, env_id
