"""GPU: the CBF condition under the policy and its state gradient (gcbf_cbf_condition, GCBFPlus.cbf_condition) against
the float64 oracle (tests/falsify_oracle.py) on the device's own topology, and the search built on it
(GCBFPlus.falsify, test.py --falsify).

Tolerances.  h to 1e-4; term to 2e-4 + 1e-3 |term| (h is divided by dt = 0.03, as the refinement's loop value).  The
worst agent must be the oracle's unless the oracle's two best eligible terms lie within that tolerance of each other or
an eligible agent's h lies within 1e-4 of 0.  grad_x to 2e-3 max |grad| (fp32 forwards and backwards of three network
passes, the 1/dt factor on both sides).  Randomly initialised networks must meet it outright; pretrained ones may instead
stay inside the float64 oracle's own ReLU-kink envelope (derivative taken as 1[x > +-1e-4]), as in
tests/test_gpu_refine.py, and such graphs must stay a minority."""
import argparse
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

from falsify_oracle import objective
from gnn_f64 import graph_of, params64
from helpers import ROOT, oracle_env, product_algo, product_env, product_obstacles, random_scene
from test_gpu_refine import shifted_relu_derivative

pytestmark = pytest.mark.gpu

CASES = [("SingleIntegrator", 4, 0.6, 2, 3), ("SingleIntegrator", 32, 1.6, 4, 4), ("DoubleIntegrator", 16, 1.2, 6, 1),
         ("DoubleIntegrator", 64, 2.4, 8, 2), ("DubinsCar", 8, 1.0, 4, 5), ("DubinsCar", 48, 2.0, 6, 6),
         ("LinearDrone", 6, 0.8, 4, 6), ("LinearDrone", 64, 1.6, 6, 7)]
G = 3
H_TOL = 1e-4
GRAD_TOL = 2e-3
KINK_DELTA = 1e-4


def _term_tol(t):
    return 2e-4 + 1e-3 * np.abs(t)


def _setup(env_id, N, G, area, n_obs, seed, pretrained):
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 64
    algo = product_algo(env, env_id if pretrained else None, seed=3)
    pobs = product_obstacles(env_id, obs)
    return env, algo, agent, goal, pobs


def _graph(env, agent, goal, pobs):
    return env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)


def _center_cbf(algo, graph):
    """A xavier CBF (zero biases) may be negative on every agent, leaving no agent to differentiate: shift its output
    bias by the median pre-activation, so that about half of the agents have h >= 0."""
    h = algo.get_cbf(graph).double().clamp(-0.999999, 0.999999)
    tree = algo.cbf_params.to_tree()
    tree["params"]["Dense_0"]["bias"] = np.asarray(tree["params"]["Dense_0"]["bias"]) - np.float32(
        float(torch.atanh(h).median()))
    algo.cbf_params.from_tree(tree)


@pytest.mark.parametrize("env_id,N,area,n_obs,seed", CASES)
@pytest.mark.parametrize("pretrained", [True, False])
def test_condition_and_gradient_match_float64(env_id, N, area, n_obs, seed, pretrained, gemm_path):
    """h, term and the worst agent of every graph, and d J / dx: the chain through cbf(g'), the Euler step and u_ref,
    the actor's data-only backward with the edge-state output (upstream d J / d pi) and the CBF's on g."""
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, seed, pretrained)
    graph = _graph(env, agent, goal, pobs)
    if not pretrained:
        _center_cbf(algo, graph)
    h, term, worst, grad = algo.cbf_condition(graph, with_grad=True)
    h2, term2, worst2 = algo.cbf_condition(graph)
    torch.cuda.synchronize()
    graph.check_overflow()
    # the forward-only call runs the same launches up to the selection
    assert torch.equal(h, h2) and torch.equal(term, term2) and torch.equal(worst, worst2)
    oenv = oracle_env(env_id, N, area, n_obs, dtype=torch.float64)
    cp, ap = params64(algo.cbf_params), params64(algo.actor_net_params)
    h, term, worst, grad = (t.cpu().double() for t in (h, term, worst, grad))
    n_kink = n_checked = 0
    for g in range(G):
        og = graph_of(oenv, graph, g, clip_all=0)
        x = torch.from_numpy(agent[g]).double()
        o = objective(oenv, cp, ap, og, x, algo.alpha)
        np.testing.assert_allclose(h[g].numpy(), o["h"].numpy(), atol=H_TOL, rtol=0, err_msg=f"h, graph {g}")
        ot = o["term"].numpy()
        assert (np.isnan(term[g].numpy()) == np.isnan(ot)).all()
        fin = np.isfinite(ot)
        assert (np.abs(term[g].numpy()[fin] - ot[fin]) <= _term_tol(ot[fin])).all(), (g, term[g], ot)
        w = int(worst[g])
        if w != o["worst"]:
            elig = (o["h"] >= 0).numpy() & fin
            top = np.sort(ot[elig])[::-1]
            tie = len(top) > 1 and top[0] - top[1] <= 2 * _term_tol(top[0])
            near0 = bool((np.abs(o["h"].numpy()[fin]) < H_TOL).any())
            assert tie or near0, (g, w, o["worst"], top[:3])
            continue
        if w < 0:
            assert float(grad[g].abs().max()) == 0.0
            continue
        n_checked += 1
        scale = float(o["grad"].abs().max())
        err = (grad[g] - o["grad"]).abs()
        if float(err.max()) <= GRAD_TOL * scale:
            continue
        assert pretrained, (g, float(err.max()) / scale, "a randomly initialised network has no ReLU ties")
        with shifted_relu_derivative(+KINK_DELTA):
            hi = objective(oenv, cp, ap, og, x, algo.alpha, agent=w)["grad"]
        with shifted_relu_derivative(-KINK_DELTA):
            lo = objective(oenv, cp, ap, og, x, algo.alpha, agent=w)["grad"]
        slack = 3.0 * ((hi - o["grad"]).abs() + (lo - o["grad"]).abs())
        assert float((err - slack).max()) <= GRAD_TOL * scale, (g, float(err.max()) / scale)
        n_kink += 1
    assert n_checked > 0, "no graph had a worst agent: the gradient was not exercised"
    assert n_kink <= max(1, G // 3)


def _verify_public(algo, env, states, goal, obs):
    """h and term through the public path: env.get_graph, get_cbf, act, env.forward_graph, get_cbf."""
    gr = env.get_graph(states, goal, obs)
    h = algo.get_cbf(gr).squeeze(-1)
    hn = algo.get_cbf(env.forward_graph(gr, algo.act(gr))).squeeze(-1)
    return h, -((hn - h) / env.dt) - algo.alpha * h


def test_search_improves_reverifies_and_is_deterministic():
    env_id, N, Gs, area, n_obs, seed = "DoubleIntegrator", 16, 12, 1.4, 6, 11
    env, algo, agent, goal, pobs = _setup(env_id, N, Gs, area, n_obs, seed, True)
    x = torch.from_numpy(agent).cuda()
    gl = torch.from_numpy(goal).cuda()
    before = (algo.cbf_params.flat.clone(), algo.actor_net_params.flat.clone())
    r = algo.falsify(x, gl, pobs, 12)
    r2 = algo.falsify(x, gl, pobs, 12)
    torch.cuda.synchronize()
    assert torch.equal(before[0], algo.cbf_params.flat) and torch.equal(before[1], algo.actor_net_params.flat)
    for k, v in r.items():
        if torch.is_tensor(v):
            assert torch.equal(v.view(torch.int32) if v.dtype == torch.float32 else v,
                               r2[k].view(torch.int32) if v.dtype == torch.float32 else r2[k]), k
        else:
            assert v == r2[k], k
    assert bool((r["J"] >= r["J0"]).all())
    assert bool((r["iter"] >= 0).all()) and bool((r["iter"] < 12).all())
    # the start is iteration 0 of the search: J0 is the condition at the given states
    h0, t0, w0 = algo.cbf_condition(env.get_graph(x, gl, pobs))
    from gcbfplus_b200.algo.falsify import worst_value
    assert torch.equal(worst_value(t0, w0), r["J0"])
    # every counterexample re-verifies through the public path (which runs the folded inference forward: the values
    # agree to rounding)
    h, t = _verify_public(algo, env, r["agent"], gl, pobs)
    n_cex = 0
    for g in range(Gs):
        w = int(r["worst"][g])
        if w < 0:
            continue
        assert abs(float(h[g, w]) - float(r["h"][g, w])) <= H_TOL
        assert abs(float(t[g, w]) - float(r["term"][g, w])) <= _term_tol(float(r["term"][g, w]))
        if float(r["J"][g]) > 1e-3 and float(r["h"][g, w]) > H_TOL:
            assert float(h[g, w]) >= 0 and float(t[g, w]) > 0, (g, w)
            n_cex += 1
    print(f"counterexamples: {n_cex} of {Gs} graphs; J0 > 0 in {int((r['J0'] > 0).sum())}")
    fs0 = int((env.unsafe_mask(env.get_graph(x, gl, pobs)) & (h0 >= 0)).sum())
    assert r["false_safe0"] == fs0


def test_multi_layer_networks_are_rejected():
    from gcbfplus_b200.algo import make_algo
    env_id, N, Gs = "DoubleIntegrator", 4, 2
    env = product_env(env_id, N, 2.0, 0)
    deep = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, gnn_layers=2, seed=1)
    agent, goal, _ = random_scene(env_id, N, Gs, 2.0, 0, seed=1)
    graph = _graph(env, agent, goal, None)
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        deep.cbf_condition(graph, with_grad=True)
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        deep.falsify(graph.agent, graph.goal, None, 3)


def test_test_py_falsify_end_to_end(tmp_path, capsys):
    """A run saved from the pretrained DoubleIntegrator npz, searched by test.py --path --falsify 20."""
    import yaml
    env_id, N = "DoubleIntegrator", 6
    env = product_env(env_id, N, 1.5, 2)
    algo = product_algo(env, env_id)
    algo.save(str(tmp_path / "models"), 0)
    cfg = argparse.Namespace(env=env_id, num_agents=N, algo="gcbf+", buffer_size=algo.buffer_size, **algo.config)
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_falsify_gpu", os.path.join(ROOT, "test.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    args = cli.build_test_parser().parse_args(["--path", str(tmp_path), "--area-size", "1.5", "--obs", "2", "--epi", "3",
                                               "--max-step", "24", "--falsify", "20", "--no-video"])
    cli.test(args)
    out = capsys.readouterr().out
    print(out)
    assert "falsify: 75 graphs searched (20 iterations)" in out
    z = np.load(tmp_path / "falsify" / "step0.npz")
    assert z["agent"].shape == (75, N, 4) and z["J"].shape == (75,)
    assert (z["J"] >= z["J0"]).all()
