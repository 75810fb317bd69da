"""CPU: test.py's --online-refine flag handling, and the loop semantics of the refinement oracle
(tests/refine_oracle.py, gcbf.py:161-201): the stopping test reads the value before the update, the first iteration
always runs, a NaN value ends the loop, and max_iter caps it."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, oracle_env, oracle_params


def _test_cli():
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_refine", os.path.join(ROOT, "test.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    from train import build_parser
    return mod, lambda argv: build_parser(mod.FLAGS).parse_args(argv)


def test_online_refine_flag_parsing_and_rejections():
    cli, parse = _test_cli()
    args = parse(["--path", "runs/x", "--area-size", "2.0", "--online-refine"])
    assert args.online_refine and args.path == "runs/x"
    cli.check_refine_flags(args)                                     # a trained run: accepted
    assert not parse(["--path", "runs/x", "--area-size", "2.0"]).online_refine
    for argv, what in ((["--env", "DoubleIntegrator", "--u-ref"], "--u-ref"),
                       (["--env", "DoubleIntegrator", "--algo", "dec_share_cbf"], "dec_share_cbf"),
                       (["--env", "DoubleIntegrator", "--algo", "centralized_cbf"], "centralized_cbf"),
                       (["--env", "DoubleIntegrator"], "--path"),
                       (["--path", "runs/x", "--u-ref"], "--u-ref")):
        with pytest.raises(SystemExit, match=what):
            cli.check_refine_flags(parse(argv + ["--area-size", "2.0", "--online-refine"]))
    with pytest.raises(SystemExit, match="--u-ref"):          # rejected before anything is built or loaded
        cli.test(parse(["--env", "DoubleIntegrator", "--u-ref", "--area-size", "2.0", "--online-refine"]))


def _scripted(monkeypatch, vals):
    """Replace the loop value by a scripted sequence with gradient c = (1, 2, ...) per action entry."""
    import refine_oracle
    seq = iter(vals)

    def fake(env, cbf_p, g, h, a, alpha):
        c = torch.arange(1, a.numel() + 1, dtype=a.dtype).reshape(a.shape)
        lin = (a * c).sum()
        return lin - lin.detach() + torch.tensor(next(seq), dtype=a.dtype)
    monkeypatch.setattr(refine_oracle, "refine_value", fake)
    return refine_oracle


def _graph(env_id="DoubleIntegrator", N=3, dtype=torch.float64):
    env = oracle_env(env_id, N, 2.0, 0, dtype=dtype)
    actor_p, cbf_p = oracle_params(env_id, dtype)
    agent = torch.tensor([[0.2, 0.2, 0.0, 0.0], [1.0, 1.0, 0.1, 0.0], [1.7, 0.3, 0.0, -0.1]], dtype=dtype)
    goal = torch.tensor([[1.5, 1.5, 0, 0], [0.2, 1.8, 0, 0], [0.4, 0.4, 0, 0]], dtype=dtype)
    return env, actor_p, cbf_p, agent, goal


@pytest.mark.parametrize("vals,max_iter,want", [([0.5, 0.2, 0.0, 0.7], 30, 3),     # stops after the first 0
                                                 ([0.0], 30, 1),                   # mandatory first step
                                                 ([0.5, float("nan"), 0.3], 30, 2),  # NaN > 0 is False
                                                 ([0.5] * 10, 4, 4)])              # cap
def test_oracle_loop_semantics(monkeypatch, vals, max_iter, want):
    env, actor_p, cbf_p, agent, goal = _graph()
    g = env.sparsify(env.get_graph(agent, goal, None))
    ro = _scripted(monkeypatch, vals)
    a0 = ro.refine_oracle(env, cbf_p, actor_p, g, max_iter=1, lr=0.0)["action"]
    ro = _scripted(monkeypatch, vals)
    out = ro.refine_oracle(env, cbf_p, actor_p, g, lr=0.1, max_iter=max_iter)
    assert out["iters"] == want
    np.testing.assert_equal(out["values"], vals[:want])
    # every iteration applies its update, the last one included (gradient c per entry, value-independent here)
    c = torch.arange(1, a0.numel() + 1, dtype=a0.dtype).reshape(a0.shape)
    torch.testing.assert_close(out["action"], a0 - 0.1 * c * want, rtol=0, atol=1e-12)


def test_oracle_nan_u_ref_stops_after_one_iteration():
    """An agent exactly at its goal has u_ref = NaN (0 / 0 in the error clip): its NaN reaches the value."""
    env, actor_p, cbf_p, agent, goal = _graph()
    from refine_oracle import refine_oracle
    goal[1] = agent[1].clone()
    agent[1, 2:] = 0.0
    goal[1, 2:] = 0.0
    g = env.sparsify(env.get_graph(agent, goal, None))
    out = refine_oracle(env, cbf_p, actor_p, g)
    assert torch.isnan(out["u_ref"][1]).all()
    assert out["iters"] == 1 and np.isnan(out["values"][0])


def test_oracle_safe_graph_keeps_u_ref():
    """Agents far apart and from any obstacle: v_ref = 0 everywhere, so a = u_ref; the one mandatory step sees value
    0 and a zero gradient."""
    env, actor_p, cbf_p, agent, goal = _graph()
    from refine_oracle import refine_oracle
    g = env.sparsify(env.get_graph(agent, goal, None))
    out = refine_oracle(env, cbf_p, actor_p, g)
    assert not bool(out["sel"].any()), out["sel_term"]
    assert out["iters"] == 1 and out["values"] == [0.0]
    assert torch.equal(out["action"], out["u_ref"])
