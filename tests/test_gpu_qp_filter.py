"""GPU: the learned-CBF QP safety filter -- gcbf_qp_filter, GCBFPlus.safety_filter and the rollout engine's actor_qp /
u_ref_qp policies -- on both GEMM paths.

* With a NULL nominal the filter is the labels' QP, bit for bit; with the u_ref that gcbf_act writes it agrees within
  1e-6 (whether those bits are identical too is printed).
* With random nominals inside and outside the u_lim box, the device solution matches the float64 dual solve of the
  oracle (oracle/qp.py) on the same assembled Lg_h / b to the labels' tolerance and satisfies the QP's KKT conditions;
  the scenes have binding CBF rows, so the check is not just u == u_nom.
* The rollout policies build canonical graphs: every recorded step equals the labels / the filter evaluated on the graph
  env.get_graph rebuilds from the recorded state, bit for bit; captured, eager and repeated rollouts give the same bits.
"""
import argparse
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, product_algo, product_env, product_obstacles, random_scene

pytestmark = pytest.mark.gpu

CASES = [("SingleIntegrator", 8, 3, 0.9, 4, 3), ("DoubleIntegrator", 16, 3, 1.6, 8, 1),
         ("DubinsCar", 12, 2, 1.4, 6, 5), ("LinearDrone", 10, 2, 1.0, 4, 6)]


def _scene(env_id, N, G, area, n_obs, seed, vel_scale=0.4):
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=seed, vel_scale=vel_scale)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 64
    algo = product_algo(env, env_id)
    pobs = product_obstacles(env_id, obs)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    return env, algo, graph, (agent, goal, pobs)


def _bits_equal(x, y):
    return torch.equal(x.contiguous().view(torch.int32), y.contiguous().view(torch.int32))


def _abi_filter(env, algo, graph, u_nom, max_iter, tol):
    """gcbf_qp_filter through the C ABI (u_nom may be None: NULL), on the workspace safety_filter / qp_labels cache."""
    from gcbfplus_b200 import _lib
    G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
    d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
    ws = algo._qp_ws["ws"]
    u = torch.empty(G, N, nu, dtype=torch.float32, device="cuda")
    aux = torch.empty(G, N, 2, dtype=torch.float32, device="cuda")
    iters = torch.empty(G, dtype=torch.int32, device="cuda")
    rc = env.lib.gcbf_qp_filter(C.byref(d), float(algo.alpha), 1 if _lib.USE_TC else 0, max_iter, tol,
                                _lib.ptr(algo.cbf_params.flat), _lib.ptr(graph.agent), _lib.ptr(graph.goal),
                                _lib.ptr(graph.hits), _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg),
                                _lib.ptr(graph.edge_recv), _lib.ptr(graph.edge_src), _lib.ptr(graph.counters),
                                _lib.ptr(u_nom), _lib.ptr(u), _lib.ptr(aux), _lib.ptr(iters), _lib.ptr(ws), ws.numel(),
                                env._stream())
    _lib.check(rc, "gcbf_qp_filter")
    return u, aux, iters


@pytest.mark.parametrize("env_id,N,G,area,n_obs,seed", CASES)
def test_null_nominal_is_the_labels(env_id, N, G, area, n_obs, seed, gemm_path):
    from gcbfplus_b200.algo.train import QP_MAX_ITER, QP_TOL, batch_u_ref, qp_labels
    env, algo, graph, _ = _scene(env_id, N, G, area, n_obs, seed)
    u0, aux0, it0 = qp_labels(algo, graph, params=algo.cbf_params, with_aux=True)
    u1, aux1, it1 = _abi_filter(env, algo, graph, None, QP_MAX_ITER, QP_TOL)
    torch.cuda.synchronize()
    graph.check_overflow()
    assert _bits_equal(u0, u1) and _bits_equal(aux0, aux1) and torch.equal(it0, it1 & 0x3FFFFFFF)
    u_ref = batch_u_ref(algo, {"agent": graph.agent, "goal": graph.goal})
    u2, r2, it2 = algo.safety_filter(graph, u_ref, return_info=True)
    torch.cuda.synchronize()
    err = float((u2 - u0).abs().max())
    print(f"{env_id} {gemm_path}: u_nom = u_ref from gcbf_act vs NULL: max |du| {err:.3g}, bit-identical "
          f"{_bits_equal(u2, u0) and _bits_equal(r2, aux0[..., 1])}")
    assert err <= 1e-6
    torch.testing.assert_close(r2, aux0[..., 1], rtol=0, atol=1e-6)


@pytest.mark.parametrize("env_id,N,G,area,n_obs,seed", CASES)
def test_random_nominals_match_oracle(env_id, N, G, area, n_obs, seed, gemm_path):
    from oracle import qp
    from test_gpu_qp import _qp_from_device
    env, algo, graph, _ = _scene(env_id, N, G, area, n_obs, seed)
    nu = env.action_dim
    u_lim = float(env.action_lim()[1][0])
    rng = np.random.Generator(np.random.PCG64(seed + 100))
    # half the entries inside the box, half outside it (up to twice the limit)
    u_nom = rng.uniform(-2 * u_lim, 2 * u_lim, size=(G, N, nu)).astype(np.float32)
    u_dev, r_dev, iters = algo.safety_filter(graph, torch.from_numpy(u_nom).cuda(), max_iter=20000, tol=1e-6,
                                             return_info=True)
    torch.cuda.synchronize()
    graph.check_overflow()
    assert int(iters.max()) < 20000, "dual iteration did not reach its tolerance"
    dev = _qp_from_device(env, algo._qp_ws["ws"], graph, N, nu)
    u_dev = u_dev.cpu().numpy().astype(np.float64)
    r_dev = r_dev.cpu().numpy().astype(np.float64)
    n_active = n_moved = n_box = 0
    for g in range(G):
        np.testing.assert_array_equal(dev[g]["u_ref"], u_nom[g].reshape(-1).astype(np.float64))   # UR = u_nom
        u, r, lam, _ = qp.solve_qp_dual(dev[g]["Lg"], dev[g]["b"], dev[g]["u_ref"], u_lim)
        np.testing.assert_allclose(u_dev[g].reshape(-1), u, atol=5e-4, rtol=0)
        np.testing.assert_allclose(r_dev[g], r, atol=1e-3, rtol=1e-3)
        kkt = qp.kkt_residual(dev[g]["Lg"], dev[g]["b"], dev[g]["u_ref"], u_lim, u_dev[g].reshape(-1), r_dev[g], lam)
        assert kkt["stationarity_u"] < 1e-4 and kkt["primal"] < 1e-3 and kkt["dual"] == 0.0, kkt
        n_active += int((lam > 0).sum())
        n_moved += int((np.abs(u_dev[g].reshape(-1) - np.clip(u_nom[g].reshape(-1), -u_lim, u_lim)) > 1e-3).sum())
        n_box += int((np.abs(u_dev[g]) == np.float32(u_lim)).sum())
    assert n_active > 0 and n_moved > 0, "no CBF constraint binds: the test would only check u == clip(u_nom)"
    assert n_box > 0, "no action at the box limit"


def _rollout(env, algo, policy, E, T, agent0, goal, pobs, use_cuda_graph=True):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    eng = RolloutEngine(env, E, T=T, policy=policy, use_cuda_graph=use_cuda_graph)
    eng.set_params(algo.actor_params)
    eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
    eng.set_initial(torch.as_tensor(agent0).cuda(), torch.as_tensor(goal).cuda(), pobs)
    eng.run()
    torch.cuda.synchronize()
    ch = eng.chains[0]
    return eng, [eng.agent.clone(), eng.actions.clone(), ch.qp_iters.clone(), ch.qp_nominal.clone(), ch.qp_aux.clone()]


@pytest.mark.parametrize("env_id,N,area,n_obs,seed", [("DoubleIntegrator", 8, 1.5, 2, 4), ("SingleIntegrator", 8, 1.5, 2, 8)])
def test_rollout_steps_equal_filter_on_rebuilt_graphs(env_id, N, area, n_obs, seed, gemm_path):
    """Each recorded state's graph rebuilt by env.get_graph: u_ref_qp's action equals qp_labels on it bit for bit;
    actor_qp's equals safety_filter on it with the recorded nominal bit for bit, and that nominal equals algo.act
    (the unfolded forward, where the rollout runs the folded inference network) to rounding."""
    from gcbfplus_b200.algo.train import qp_labels
    E, T = 3, 24
    env, algo, _, (agent, goal, pobs) = _scene(env_id, N, E, area, n_obs, seed, vel_scale=0.0)
    n_binding = 0
    for policy in ("u_ref_qp", "actor_qp"):
        eng, (states, actions, iters, nominal, aux) = _rollout(env, algo, policy, E, T, agent, goal, pobs)
        st = eng.qp_stats()
        assert st["solves"] == E * T
        print(f"{env_id} {gemm_path} {policy}: {st}")
        worst = 0.0
        for t in range(T):
            g = env.get_graph(states[t], eng.goal, pobs)
            assert _bits_equal(g.hits, eng.hits[t])
            if policy == "u_ref_qp":
                u, a2, it = qp_labels(algo, g, params=algo.cbf_params, with_aux=True)
                assert _bits_equal(u, actions[t]), t
                assert _bits_equal(a2, aux[t]) and torch.equal(it, iters[t] & 0x3FFFFFFF), t
                n_binding += int((a2[..., 0] > 0).sum())
            else:
                u, r, it = algo.safety_filter(g, nominal[t], return_info=True)
                assert _bits_equal(u, actions[t]) and _bits_equal(r, aux[t][..., 1]), t
                act = algo.act(g)
                torch.testing.assert_close(act, nominal[t], rtol=0, atol=1e-5)
                worst = max(worst, float((algo.safety_filter(g, act) - actions[t]).abs().max()))
        if policy == "actor_qp":
            print(f"{env_id} {gemm_path}: max |safety_filter(g, algo.act(g)) - action| = {worst:.3g}")
            assert worst <= 1e-3
    torch.cuda.synchronize()
    assert n_binding > 0, "no CBF row bound along the u_ref_qp rollout"


@pytest.mark.parametrize("policy", ["actor_qp", "u_ref_qp"])
def test_captured_eager_and_repeated_rollouts_agree(policy, gemm_path):
    env_id, N, E, T, area, n_obs = "DoubleIntegrator", 16, 3, 16, 1.6, 6
    env, algo, _, (agent, goal, pobs) = _scene(env_id, N, E, area, n_obs, 2)
    eng, first = _rollout(env, algo, policy, E, T, agent, goal, pobs)
    assert eng._graph is not None
    eng.run()                                      # a replay of the captured graph
    torch.cuda.synchronize()
    ch = eng.chains[0]
    again = [eng.agent, eng.actions, ch.qp_iters, ch.qp_nominal, ch.qp_aux]
    _, eager = _rollout(env, algo, policy, E, T, agent, goal, pobs, use_cuda_graph=False)
    for x, y, z in zip(first, again, eager):
        assert _bits_equal(x, y) and _bits_equal(x, z)
    # the settings are baked into the captured launches: a new alpha drops the graph, the same one keeps it
    eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
    assert eng._graph is not None
    eng.set_cbf_params(algo.cbf_params, alpha=2 * algo.alpha)
    assert eng._graph is None


def test_refusals():
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env_id, N, G = "DoubleIntegrator", 4, 2
    env = product_env(env_id, N, 2.0, 0)
    deep = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, gnn_layers=2, seed=1)
    shallow = product_algo(env, env_id)
    agent, goal, _ = random_scene(env_id, N, G, 2.0, 0, seed=1)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), None)
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        deep.safety_filter(graph)
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        shallow.safety_filter(graph, cbf_params=deep.cbf_params)
    with pytest.raises(ValueError, match="shape"):
        shallow.safety_filter(graph, torch.zeros(G, N + 1, env.action_dim, device="cuda"))
    for policy in ("actor_qp", "u_ref_qp"):
        with pytest.raises(ValueError, match="persistent"):
            RolloutEngine(env, G, T=4, policy=policy, persistent=True)
        eng = RolloutEngine(env, G, T=4, policy=policy)
        assert not eng.persistent
        with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
            eng.set_cbf_params(deep.cbf_params)
        with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
            eng.set_params(deep.actor_params)
        eng.set_params(shallow.actor_params)
        eng.set_initial(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), None)
        with pytest.raises(RuntimeError, match="set_cbf_params"):
            eng.run()
    eng = RolloutEngine(env, G, T=4, policy="actor")
    with pytest.raises(RuntimeError, match="qp_stats"):
        eng.qp_stats()
    with pytest.raises(RuntimeError, match="set_cbf_params"):
        eng.set_cbf_params(shallow.cbf_params)
    # more agents than the solver's shared-memory layout allows: rejected by the library
    big_env = product_env(env_id, 2049, 40.0, 0)
    big = product_algo(big_env, env_id)
    a, g, _ = random_scene(env_id, 2049, 1, 40.0, 0, seed=3)
    big_graph = big_env.get_graph(torch.from_numpy(a).cuda(), torch.from_numpy(g).cuda(), None)
    with pytest.raises(RuntimeError, match="2049 > 2048"):
        big.safety_filter(big_graph, torch.zeros(1, 2049, env.action_dim, device="cuda"))


def test_test_py_qp_filter_end_to_end(tmp_path, capsys):
    """A run saved from the pretrained DoubleIntegrator npz, evaluated by test.py --path --qp-filter (actor_qp) and
    --path --u-ref --qp-filter (u_ref_qp).  The safety rates are printed, not asserted."""
    import yaml
    env_id, N = "DoubleIntegrator", 6
    env = product_env(env_id, N, 1.5, 2)
    algo = product_algo(env, env_id)
    algo.save(str(tmp_path / "models"), 0)
    cfg = argparse.Namespace(env=env_id, num_agents=N, algo="gcbf+", buffer_size=algo.buffer_size, **algo.config)
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_qp_filter_gpu", os.path.join(ROOT, "test.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    from train import build_parser
    base = ["--path", str(tmp_path), "--area-size", "1.5", "--obs", "2", "--epi", "3", "--max-step", "24",
            "--qp-filter", "--no-video", "--log"]
    for extra in ([], ["--u-ref"]):
        cli.test(build_parser(cli.FLAGS).parse_args(base + extra))
        out = capsys.readouterr().out
        assert "QP iterations: median" in out and "of 72 solves" in out
        assert "QP filter: mean |u - u_nom|" in out and "safe_rate" in out
        with capsys.disabled():
            print(f"\ntest.py --qp-filter {' '.join(extra)}:")
            for line in out.splitlines():
                if line.startswith(("reward:", "QP ", "WARNING")):
                    print("  " + line)
    with open(tmp_path / "test_log.csv") as f:
        assert len(f.read().splitlines()) == 2
    with pytest.raises(SystemExit, match="--online-refine"):
        cli.test(build_parser(cli.FLAGS).parse_args(base + ["--online-refine"]))
