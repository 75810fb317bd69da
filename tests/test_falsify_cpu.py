"""CPU: test.py's --falsify flag handling, and the float64 oracle of the CBF-condition gradient (tests/falsify_oracle.py)
against central finite differences on a frozen topology, in all four environments."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

from falsify_oracle import features, objective, term_at
from gnn_f64 import synthetic_scene
from helpers import ENVS, ROOT, oracle_env

F64 = torch.float64


def _test_cli():
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_falsify", os.path.join(ROOT, "test.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, lambda argv: mod.build_test_parser().parse_args(argv)


def test_falsify_flag_parsing_and_rejections():
    cli, parse = _test_cli()
    args = parse(["--path", "runs/x", "--area-size", "2.0", "--falsify", "20"])
    assert args.falsify == 20
    cli.check_falsify_flags(args)
    assert parse(["--path", "runs/x", "--area-size", "2.0"]).falsify is None
    for argv, what in ((["--path", "runs/x", "--u-ref"], "--u-ref"),
                       (["--path", "runs/x", "--online-refine"], "--online-refine"),
                       (["--path", "runs/x", "--qp-filter"], "--qp-filter"),
                       (["--paths", "runs/x", "runs/y"], "--paths"),
                       (["--path", "runs/x", "--all-steps"], "--all-steps"),
                       (["--env", "DoubleIntegrator", "--algo", "dec_share_cbf"], "dec_share_cbf"),
                       (["--env", "DoubleIntegrator", "--algo", "centralized_cbf"], "centralized_cbf"),
                       (["--env", "DoubleIntegrator"], "--path"),
                       (["--path", "runs/x", "--falsify", "0"], "iterations")):
        argv = argv + ["--area-size", "2.0"] + ([] if "--falsify" in argv else ["--falsify", "5"])
        with pytest.raises(SystemExit, match=what):
            cli.check_falsify_flags(parse(argv))
        # refused before anything is built or loaded (the run directories do not exist)
        with pytest.raises(SystemExit, match=what):
            cli.test(parse(argv))


def _scene(env_id, N, seed):
    from oracle.nn import init_params, to_torch
    env = oracle_env(env_id, N, 1.0, 0, dtype=F64)
    agent, goal, hits = synthetic_scene(env_id, N, 1, 1.0, seed)
    agent[0, N - 1] += 0.05           # synthetic_scene duplicates the last agent (tied logits): separate it
    sd, pd = env.state_dim, env.pos_dim
    lidar = torch.zeros(N, env.n_hits, sd, dtype=F64)
    lidar[..., :pd] = torch.from_numpy(hits[0]).to(F64)
    x = torch.from_numpy(agent[0]).to(F64)
    g = env.sparsify(env.get_graph(x, torch.from_numpy(goal[0]).to(F64), None, lidar=lidar))
    ed = {"SingleIntegrator": 2, "LinearDrone": 6}.get(env_id, 4)
    nu = 3 if env_id == "LinearDrone" else 2
    cbf = to_torch(init_params(ed, 1, "cbf", seed * 2 + 1), F64)
    actor = to_torch(init_params(ed, nu, "actor", seed * 2 + 2), F64)
    return env, g, x, cbf, actor


@pytest.mark.parametrize("env_id", ENVS)
def test_oracle_features_are_the_graphs(env_id):
    """The oracle's re-expression of the edge features from the states reproduces get_graph's (g) and
    forward_graph's (every feature norm-clipped)."""
    env, g, x, _, _ = _scene(env_id, 6, 3)
    np.testing.assert_allclose(features(env, g, x, False).numpy(), g.edges.numpy(), rtol=0, atol=1e-12)
    clipped = env.add_edge_feats(g, g.states[:-1]).edges
    np.testing.assert_allclose(features(env, g, x, True).numpy(), clipped.numpy(), rtol=0, atol=1e-12)


@pytest.mark.parametrize("env_id", ENVS)
@pytest.mark.parametrize("seed", [1, 2])
def test_oracle_gradient_matches_central_differences(env_id, seed):
    """d term_i / dx by autograd against central differences (step 1e-6) in float64, for the agent with the largest
    finite term: within 1e-5 of max |grad| (a kink inside the difference step would be far larger)."""
    N = 5
    env, g, x, cbf, actor = _scene(env_id, N, seed)
    with torch.no_grad():
        from falsify_oracle import condition
        _, term, _ = condition(env, cbf, actor, g, x, 1.0)
    i = int(torch.argmax(torch.where(torch.isfinite(term), term, torch.full_like(term, -np.inf))))
    got = objective(env, cbf, actor, g, x, 1.0, agent=i)["grad"]
    assert float(got.abs().max()) > 0
    eps = 1e-6
    fd = torch.zeros_like(x)
    for a in range(N):
        for c in range(x.shape[1]):
            xp, xm = x.clone(), x.clone()
            xp[a, c] += eps
            xm[a, c] -= eps
            fd[a, c] = (term_at(env, cbf, actor, g, xp, 1.0, i) - term_at(env, cbf, actor, g, xm, 1.0, i)) / (2 * eps)
    err = float((got - fd).abs().max()) / float(got.abs().max())
    assert err < 1e-5, (env_id, seed, err)
