"""GPU parity of networks with more than one GNN layer (--gnn-layers > 1) against the float32 multi-layer oracle
(tests/gnn_layers_oracle.py), xavier-initialised networks: h and pi (plain and add_edge_feats graphs), the closed-loop
rollout on the step-by-step path, and a saved run evaluated by test.py --path (incl. --cbf contours)."""
import argparse
import os
import sys

import numpy as np
import pytest
import torch

from gnn_layers_oracle import net_forward
from helpers import ROOT, oracle_env, oracle_obstacles, product_env, product_obstacles, random_scene

pytestmark = pytest.mark.gpu

TOL = 3e-5   # the tensor-core path's network tolerance at one layer (test_gpu_gnn.py)
CASES = [("SingleIntegrator", 8, 3, 2.0, 4, 2), ("DoubleIntegrator", 12, 3, 2.0, 8, 2), ("DubinsCar", 12, 3, 2.5, 6, 2),
         ("LinearDrone", 10, 2, 1.5, 4, 2), ("DoubleIntegrator", 16, 2, 2.0, 6, 3)]


def _algo(env, L, seed=0):
    from gcbfplus_b200.algo import make_algo
    return make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=env.num_agents, gnn_layers=L, seed=seed)


def _oracle_params(net):
    from oracle.nn import to_torch
    return to_torch(net.to_tree(), torch.float32)


@pytest.mark.parametrize("env_id,N,G,area,n_obs,L", CASES)
def test_forward_matches_oracle(env_id, N, G, area, n_obs, L):
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=4)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 48             # dense random scenes (not collision-free)
    algo = _algo(env, L)
    assert algo.cbf_params.n_layers == L and algo.actor_params.n_layers == L
    pobs = product_obstacles(env_id, obs)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    h = algo.get_cbf(graph).cpu().numpy()
    pi = algo.get_action(graph).cpu().numpy()
    a = algo.act(graph)
    fwd = env.forward_graph(graph, a)
    h_next = algo.get_cbf(fwd).cpu().numpy()
    torch.cuda.synchronize()
    graph.check_overflow()
    oenv = oracle_env(env_id, N, area, n_obs)
    ap, cp = _oracle_params(algo.actor_params), _oracle_params(algo.cbf_params)
    packed = pobs.packed.cpu().numpy()
    n_hit_edges = 0
    with torch.no_grad():
        for g in range(G):
            og = oenv.sparsify(oenv.get_graph(torch.from_numpy(agent[g]), torch.from_numpy(goal[g]),
                                              oracle_obstacles(packed[g])))
            n_hit_edges += int((og.senders >= 2 * N).sum())
            np.testing.assert_allclose(h[g], net_forward(cp, og, "cbf").numpy(), atol=TOL, rtol=0)
            np.testing.assert_allclose(pi[g], net_forward(ap, og, "actor").numpy(), atol=TOL, rtol=0)
            ag = torch.from_numpy(a[g].cpu().numpy())
            np.testing.assert_allclose(h_next[g], net_forward(cp, oenv.forward_graph(og, ag), "cbf").numpy(), atol=TOL,
                                       rtol=0)
    assert n_hit_edges > 0
    assert np.abs(pi).max() > 1e-2


def test_strict_fp32_path_rejects_deep_networks():
    from gcbfplus_b200 import _lib
    env_id, N, G, area, n_obs = "DoubleIntegrator", 8, 1, 2.0, 2
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=1)
    env = product_env(env_id, N, area, n_obs)
    algo = _algo(env, 2)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), product_obstacles(env_id, obs))
    old = _lib.USE_TC
    _lib.USE_TC = False
    try:
        with pytest.raises(RuntimeError, match="tensor-core path only"):
            algo.get_cbf(graph)
    finally:
        _lib.USE_TC = old
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        algo.get_qp_action(graph)


def _oracle_rollout(oenv, ap, agent0, goal0, obstacles, T):
    g = oenv.get_graph(agent0, goal0, obstacles)
    states, collide, finish = [], [], []
    with torch.no_grad():
        for _ in range(T):
            a = 2 * net_forward(ap, oenv.sparsify(g), "actor") + oenv.u_ref(g.agent, g.goal)
            states.append(g.agent)
            collide.append(oenv.collision_mask(g))
            finish.append(oenv.finish_mask(g))
            g, _, _ = oenv.step(g, a)
        states.append(g.agent)
        collide.append(oenv.collision_mask(g))
        finish.append(oenv.finish_mask(g))
    return torch.stack(states).numpy(), torch.stack(collide).numpy(), torch.stack(finish).numpy()


@pytest.mark.parametrize("env_id,N,E,area,n_obs,T,L", [("DoubleIntegrator", 8, 3, 2.0, 4, 48, 2),
                                                        ("SingleIntegrator", 8, 2, 2.0, 4, 48, 2),
                                                        ("DubinsCar", 8, 2, 2.5, 4, 32, 2),
                                                        ("LinearDrone", 8, 2, 1.2, 3, 32, 2),
                                                        ("DoubleIntegrator", 8, 2, 2.0, 4, 32, 3)])
def test_rollout_matches_oracle_on_step_path(env_id, N, E, area, n_obs, T, L):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    from oracle.algo import rates
    from test_gpu_rollout import _as_rollout_result
    env = product_env(env_id, N, area, n_obs)
    g0 = env.reset(13, n_envs=E)
    algo = _algo(env, L, seed=1)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs)
    eng.set_params(algo.actor_params)
    assert eng.n_layers == L and not eng.persistent
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    first = eng.agent.clone()
    eng.run()                                   # CUDA-graph replay is bit-reproducible
    torch.cuda.synchronize()
    assert torch.equal(first, eng.agent)
    res = eng.result()
    col, fin = env.rollout_masks(_as_rollout_result(res))
    oenv = oracle_env(env_id, N, area, n_obs)
    ap = _oracle_params(algo.actor_params)
    packed = g0.obstacle.packed.cpu().numpy()
    for e in range(E):
        want, ocol, ofin = _oracle_rollout(oenv, ap, g0.agent[e].cpu(), g0.goal[e].cpu(), oracle_obstacles(packed[e]), T)
        err = np.abs(res.agent[e].cpu().numpy() - want).reshape(T + 1, -1).max(axis=1)
        assert err[1] <= 6e-6, err[:4]
        assert err[:min(T // 4, 24)].max() <= 3e-4, err
        assert err.max() <= 5e-3, err.max()
        assert rates(col[:, e].cpu().numpy(), fin[:, e].cpu().numpy()) == rates(ocol, ofin)


def test_engine_path_follows_the_current_actor():
    """An engine that ran a two-layer actor gives a one-layer actor the path (and the bits) a fresh engine gives it."""
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env_id, N, E, area, n_obs, T = "DoubleIntegrator", 8, 2, 2.0, 4, 16
    env = product_env(env_id, N, area, n_obs)
    g0 = env.reset(5, n_envs=E)
    one, two = _algo(env, 1, seed=1), _algo(env, 2, seed=1)
    fresh = RolloutEngine(env, E, T=T, n_obs=n_obs)
    fresh.set_params(one.actor_params)
    fresh.set_initial(g0.agent, g0.goal, g0.obstacle)
    fresh.run()
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    for algo in (two, one):
        eng.set_params(algo.actor_params)
        eng.run()
    torch.cuda.synchronize()
    assert eng.n_layers == 1 and eng.persistent == fresh.persistent
    assert torch.equal(eng.agent, fresh.agent) and torch.equal(eng.actions, fresh.actions)


def test_save_then_evaluate_with_test_py(tmp_path, monkeypatch):
    """A two-layer run saved in the reference layout (<dir>/models/<step>/{actor,cbf}.pkl + config.yaml) loads in
    test.py --path, rolls out and writes the --cbf contour grids."""
    import yaml
    env_id, N = "DoubleIntegrator", 4
    env = product_env(env_id, N, 2.0, 2)
    algo = _algo(env, 2, seed=3)
    algo.save(str(tmp_path / "models"), 0)
    cfg = argparse.Namespace(env=env_id, num_agents=N, algo="gcbf+", buffer_size=algo.buffer_size, **algo.config)
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    import importlib.util
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli", os.path.join(ROOT, "test.py"))
    test_cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(test_cli)
    from train import build_parser
    args = build_parser(test_cli.FLAGS).parse_args(["--path", str(tmp_path), "--area-size", "2.0", "--obs", "2",
                                                    "--epi", "2", "--max-step", "16", "--cbf", "1", "--no-video"])
    test_cli.test(args)
    out = tmp_path / "cbf_contours"
    files = sorted(os.listdir(out))
    assert files == ["epi00_agent1.npz", "epi01_agent1.npz"]
    z = np.load(out / files[0])
    assert np.isfinite(z["bb_h"]).all() and np.abs(z["bb_h"]).max() > 0
    # the loaded networks are the saved ones
    algo2 = _algo(env, 2, seed=99)
    algo2.load(str(tmp_path / "models"), 0)
    assert torch.equal(algo2.actor_params.flat, algo.actor_params.flat)
    assert torch.equal(algo2.cbf_params.flat, algo.cbf_params.flat)
