"""GPU parity of the CBF-QP baselines (csrc/cbfqp.cu) against the oracle (tests/cbfqp_oracle.py): k-nearest sets
bit-exact, h / Lie terms to fp32 rounding, QP actions against the float64 oracle solve, closed loops with identical
rates."""
import numpy as np
import pytest
import torch

import cbfqp_oracle as cq
from helpers import (ENVS, oracle_env, oracle_obstacles, product_env, product_obstacles, random_scene)

pytestmark = pytest.mark.gpu

ALGOS = ("dec_share_cbf", "centralized_cbf")


def _controller(env, algo, **kw):
    from gcbfplus_b200.algo import make_algo
    return make_algo(algo, env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=env.num_agents, **kw)


def _graph(env_id, N, G, seed):
    area = {"SingleIntegrator": 1.5, "DoubleIntegrator": 1.5, "DubinsCar": 1.5, "LinearDrone": 0.8}[env_id]
    area *= (N / 8) ** (1 / (3 if env_id == "LinearDrone" else 2))
    n_obs = 4
    env = product_env(env_id, N, area, n_obs)
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed)
    g = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), product_obstacles(env_id, obs))
    return env, g, area, n_obs


def _hit_states(env, g, gi):
    N, R, pd, sd = env.num_agents, env.n_hits, env.pos_dim, env.state_dim
    hs = torch.zeros(N, R, sd)
    hs[..., :pd] = g.hits[gi].cpu()
    return hs


def _close(got, want, what):
    scale = max(1.0, float(np.abs(want).max()))
    err = float(np.abs(got - want).max())
    assert err <= 1e-5 * scale, (what, err, scale)


@pytest.mark.parametrize("env_id", ENVS)
@pytest.mark.parametrize("N", [8, 64])
def test_pairwise_and_actions_match_oracle(env_id, N):
    G = 4
    env, g, area, n_obs = _graph(env_id, N, G, seed=100 + N)
    dec = _controller(env, "dec_share_cbf")
    cen = _controller(env, "centralized_cbf")
    pw = {k: (v.cpu().numpy() if v is not None else None) for k, v in dec.pairwise(g).items()}
    u_dec, _ = dec.get_qp_action(g)
    u_cen, _ = cen.get_qp_action(g)
    # solves that stopped at the iteration cap return the capped iterate: reported, and left out of the 1e-5 bars
    dec_ok = (dec.last_iters.reshape(G, N).cpu().numpy() & (1 << 30)) == 0
    cen_ok = (cen.last_iters.cpu().numpy() & (1 << 30)) == 0
    print(f"{env_id} N={N}: dec_share_cbf {dec.iter_stats()}, centralized_cbf {cen.iter_stats()}")
    assert dec_ok.mean() >= 0.99 and cen_ok.sum() >= G - 1
    u_dec, u_cen = u_dec.cpu().numpy(), u_cen.cpu().numpy()
    u_ref = env.u_ref(g).cpu().numpy()
    oenv = oracle_env(env_id, N, area, n_obs)
    u_lim = float(oenv.action_lim()[1][0])
    active = 0
    for gi in range(G):
        x = g.agent[gi].cpu()
        hs = _hit_states(env, g, gi)
        p = cq.pairwise(oenv, x, hs)
        np.testing.assert_array_equal(pw["idx"][gi], p["idx"].numpy())
        np.testing.assert_array_equal(pw["isobs"][gi], p["isobs"].numpy())
        _close(pw["h"][gi], p["h"].numpy(), "h")
        _close(pw["lf_h"][gi], p["lf_h"].numpy(), "Lf_h")
        _close(pw["lg_self"][gi], p["lg_self"].numpy(), "Lg_self")
        _close(pw["lg_other"][gi], p["lg_other"].numpy(), "Lg_other")
        # the float64 QP on the kernel's own data
        h, lf, ls = pw["h"][gi], pw["lf_h"][gi], pw["lg_self"][gi]
        resp = np.where(pw["isobs"][gi], np.float32(1.0), np.float32(0.5))
        b = (resp * (lf + np.float32(1.0) * h)).astype(np.float64)
        ud, _, lam, _ = cq.solve_dual_batched(ls.astype(np.float64), b, u_ref[gi].astype(np.float64), u_lim)
        np.testing.assert_allclose(u_dec[gi][dec_ok[gi]], ud[dec_ok[gi]], atol=1e-5)
        active += int((lam > 1e-9).sum())
        Lg = cq.central_from_blocks(pw["idx"][gi], pw["lg_self"][gi], pw["lg_other"][gi])
        bc = (lf + np.float32(1.0) * h).astype(np.float64).reshape(-1)
        uc, _, _, _ = cq.solve_dual_batched(Lg, bc, u_ref[gi].astype(np.float64).reshape(-1), u_lim)
        if cen_ok[gi]:
            np.testing.assert_allclose(u_cen[gi].reshape(-1), uc, atol=1e-5)
        # end to end against the oracle's float32 pipeline
        ur32 = oenv.u_ref(x, g.goal[gi].cpu())
        ue = cq.solve_dec_share(cq.dec_share_data(p, ur32), u_lim)[0]
        np.testing.assert_allclose(u_dec[gi][dec_ok[gi]], ue[dec_ok[gi]], atol=1e-4)
        ue = cq.solve_central(cq.central_data(p, ur32), u_lim)[0]
        if cen_ok[gi]:
            np.testing.assert_allclose(u_cen[gi].reshape(-1), ue, atol=1e-4)
    assert active > 0, "no CBF row is active in the scene"
    h_dec, isobs = dec.get_cbf(g)
    assert torch.equal(h_dec.cpu(), torch.from_numpy(pw["h"])) and torch.equal(isobs.cpu(), torch.from_numpy(pw["isobs"]))
    assert torch.equal(cen.get_cbf(g).cpu(), torch.from_numpy(pw["h"]))


def test_centralized_at_scale():
    """DoubleIntegrator N = 512, one graph: the 1536-row QP against the exact float64 minimiser of the kernel's own
    data, with an iteration budget the solve must converge within."""
    env, g, area, n_obs = _graph("DoubleIntegrator", 512, 1, seed=7)
    cen = _controller(env, "centralized_cbf", max_iter=200000)
    u, r = cen.get_qp_action(g)
    st = cen.iter_stats()
    print(f"centralized_cbf DoubleIntegrator N=512: {st}")
    assert st["capped"] == 0, st
    pw = {k: v.cpu().numpy() for k, v in cen.pairwise(g).items()}
    Lg = cq.central_from_blocks(pw["idx"][0], pw["lg_self"][0], pw["lg_other"][0])
    b = (pw["lf_h"][0] + np.float32(1.0) * pw["h"][0]).astype(np.float64).reshape(-1)
    ur = env.u_ref(g).cpu().numpy().astype(np.float64).reshape(-1)
    u_lim = float(env.action_lim()[1][0])
    uo, ro, lam, its = cq.solve_dual_batched(Lg, b, ur, u_lim)
    assert (lam > 1e-9).any()
    slack = -(Lg @ uo) - ro - b
    assert max(float(np.maximum(slack, 0).max()), float(np.abs(lam * slack).max())) <= 1e-8
    np.testing.assert_allclose(u.cpu().numpy().reshape(-1), uo, atol=1e-5)
    np.testing.assert_allclose(r.cpu().numpy().reshape(-1), ro, atol=1e-4)


def test_qp_stats_reports_capped_solves():
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env = product_env("DoubleIntegrator", 16, 1.5, 4)
    g0 = env.reset(3, n_envs=2)
    for algo in ALGOS:
        ctl = _controller(env, algo, max_iter=1)
        eng = RolloutEngine(env, 2, T=8, n_obs=4, policy=ctl)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        eng.run()
        st = eng.qp_stats()
        assert st["iters_max"] == 1 and st["capped"] > 0, st
        assert st["solves"] == 8 * (2 * 16 if algo == "dec_share_cbf" else 2)


def _as_result(res):
    from gcbfplus_b200.env.base import RolloutResult
    g = {"agent": res.agent.transpose(0, 1).contiguous(), "goal": res.goal, "hits": res.hits.transpose(0, 1).contiguous(),
         "obstacle": res.obstacle}
    return RolloutResult(g, res.actions.transpose(0, 1), res.rewards.transpose(0, 1), res.costs.transpose(0, 1),
                         res.dones.transpose(0, 1), {})


def test_nan_u_ref_at_goal():
    """An agent exactly at its goal has a NaN u_ref (its normalised goal error is 0 / 0).  Both baselines carry it
    through the solve as 0 and return NaN exactly in that agent's NaN u_ref components, as the reference's solve does;
    every other agent's action stays finite."""
    env_id, N, G, area, n_obs = "DoubleIntegrator", 8, 2, 1.5, 4
    env = product_env(env_id, N, area, n_obs)
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=11)
    agent[0, 3] = goal[0, 3]
    g = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), product_obstacles(env_id, obs))
    nan_ref = torch.isnan(env.u_ref(g)).cpu()
    assert nan_ref[0, 3].all() and int(nan_ref.sum()) == nan_ref[0, 3].numel()
    for algo in ALGOS:
        u = _controller(env, algo).get_qp_action(g)[0].cpu()
        assert torch.equal(torch.isnan(u), nan_ref), algo
        assert bool(torch.isfinite(u[~nan_ref]).all()), algo


@pytest.mark.parametrize("algo", ALGOS)
@pytest.mark.parametrize("env_id", ["SingleIntegrator", "DoubleIntegrator", "DubinsCar"])
def test_closed_loop_matches_oracle(env_id, algo):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    from oracle.algo import rates
    N, E, T, area, n_obs = 8, 4, 64, 2.0, 4
    env = product_env(env_id, N, area, n_obs)
    g0 = env.reset(21, n_envs=E)
    ctl = _controller(env, algo)
    enable_stop = getattr(env, "enable_stop", True)
    assert enable_stop == (algo != "dec_share_cbf" or env_id != "DubinsCar")
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, policy=ctl)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    first = eng.agent.clone()
    eng.run()                                     # CUDA-graph replay is bit-reproducible
    torch.cuda.synchronize()
    assert torch.equal(first, eng.agent)
    st = eng.qp_stats()
    print(f"{env_id} {algo} closed loop: {st}")
    res = eng.result()
    col, fin = env.rollout_masks(_as_result(res))
    oenv = oracle_env(env_id, N, area, n_obs)
    packed = g0.obstacle.packed.cpu().numpy()
    for e in range(E):
        ref = cq.rollout_controller(oenv, lambda g: cq.act(oenv, g, algo), g0.agent[e].cpu(), g0.goal[e].cpu(),
                                    oracle_obstacles(packed[e]), T=T, enable_stop=enable_stop)
        got = res.agent[e].cpu().numpy()
        want = ref["states"].numpy()
        err = np.abs(got - want).reshape(T + 1, -1).max(axis=1)
        assert err[1] <= 6e-6, err[:4]
        assert err[:16].max() <= 3e-4, err[:16].max()
        assert err.max() <= 5e-3, err.max()
        got_rates = rates(col[:, e].cpu().numpy(), fin[:, e].cpu().numpy())
        want_rates = rates(ref["collision"].numpy(), ref["finish"].numpy())
        assert got_rates == want_rates, (got_rates, want_rates)


def test_dubins_stop_mask_switch():
    """env.step applies the DubinsCar stop mask until DecShareCBF turns it off; the other step modes are unchanged."""
    env = product_env("DubinsCar", 4, 2.0, 0)
    agent = torch.tensor([[[0.5, 0.5, 0.3, 0.8], [1.5, 1.5, 0.0, 0.5], [0.2, 1.5, 1.0, 0.4], [1.5, 0.2, 2.0, 0.3]]]).cuda()
    goal = agent.clone()
    goal[0, 0, 0] += 0.01                         # agent 0 within half a radius of its goal: stopped
    goal[0, 1:, :2] += 0.7
    g = env.get_graph(agent, goal, None)
    a = torch.full((1, 4, 2), 0.1, device="cuda")
    stopped = env.step(g, a).graph.agent
    assert torch.equal(stopped[0, 0], agent[0, 0])
    u_ref_next = env._dynamics(g, None, None, 2)[1]
    via_input = env._dynamics(g, env.u_ref(g), None, 1)[1]
    assert torch.equal(u_ref_next, via_input)
    _controller(env, "dec_share_cbf")
    assert env.enable_stop is False
    moving = env.step(g, a).graph.agent
    assert not torch.equal(moving[0, 0], agent[0, 0])
    assert torch.equal(moving[0, 1:], stopped[0, 1:])
    with pytest.raises(ValueError):
        from gcbfplus_b200.trainer.rollout import RolloutEngine
        RolloutEngine(env, 1, T=4, n_obs=0, policy="u_ref")
