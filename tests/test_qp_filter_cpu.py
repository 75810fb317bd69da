"""CPU: test.py's --qp-filter flag handling, and the oracle's dual QP solve (oracle/qp.py) with a nominal action in
place of u_ref -- the QP the safety filter (gcbf_qp_filter, GCBFPlus.safety_filter) solves."""
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

from helpers import ROOT, oracle_env, oracle_params


def _test_cli():
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_qp_filter", os.path.join(ROOT, "test.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    from train import build_parser
    return mod, lambda argv: build_parser(mod.FLAGS).parse_args(argv)


def test_qp_filter_flag_parsing_and_rejections():
    cli, parse = _test_cli()
    for argv in (["--path", "runs/x"], ["--path", "runs/x", "--u-ref"]):
        args = parse(argv + ["--area-size", "2.0", "--qp-filter"])
        assert args.qp_filter and args.path == "runs/x"
        cli.check_qp_filter_flags(args)                              # a trained run, policy or u_ref: accepted
        cli.check_refine_flags(args)
    assert not parse(["--path", "runs/x", "--area-size", "2.0"]).qp_filter
    for argv, what in ((["--path", "runs/x", "--online-refine"], "--online-refine"),
                       (["--env", "DoubleIntegrator", "--algo", "dec_share_cbf"], "dec_share_cbf"),
                       (["--env", "DoubleIntegrator", "--algo", "centralized_cbf"], "centralized_cbf"),
                       (["--path", "runs/x", "--algo", "centralized_cbf"], "centralized_cbf"),
                       (["--env", "DoubleIntegrator"], "--path"),
                       (["--env", "DoubleIntegrator", "--u-ref"], "--path")):
        with pytest.raises(SystemExit, match=what):
            cli.check_qp_filter_flags(parse(argv + ["--area-size", "2.0", "--qp-filter"]))
    # rejected before anything is built or loaded (the run directory does not exist)
    for argv in (["--path", "runs/missing", "--online-refine"], ["--env", "DoubleIntegrator", "--u-ref"]):
        with pytest.raises(SystemExit):
            cli.test(parse(argv + ["--area-size", "2.0", "--qp-filter"]))


def _qp_data(alpha=1.0):
    from oracle import qp
    dt = torch.float64
    env = oracle_env("DoubleIntegrator", 4, 2.0, 0, dtype=dt)
    _, cbf_p = oracle_params("DoubleIntegrator", dt)
    agent = torch.tensor([[0.20, 0.20, 0.30, 0.10], [0.35, 0.22, -0.30, 0.0], [1.0, 1.0, 0.1, 0.0],
                          [1.7, 0.3, 0.0, -0.1]], dtype=dt)
    goal = torch.tensor([[1.5, 1.5, 0, 0], [0.1, 1.8, 0, 0], [0.2, 1.8, 0, 0], [0.4, 0.4, 0, 0]], dtype=dt)
    g = env.sparsify(env.get_graph(agent, goal, None))
    return env, cbf_p, g, qp.qp_data(env, cbf_p, g, alpha)


def test_oracle_nominal_u_ref_is_get_qp_action():
    from oracle import qp
    env, cbf_p, g, d = _qp_data()
    u0, r0, lam0, _ = qp.get_qp_action(env, cbf_p, g)
    u, r, lam, _ = qp.solve_qp_dual(d["Lg_h"], d["b"], d["u_ref"], d["u_lim"])
    np.testing.assert_array_equal(u.reshape(u0.shape), u0)
    np.testing.assert_array_equal(r, r0)
    np.testing.assert_array_equal(lam, lam0)
    # the two close agents' rows bind: the scene filters u_ref, it does not pass it through
    assert (lam0 > 0).any() and np.abs(u0.reshape(-1) - np.clip(d["u_ref"], -d["u_lim"], d["u_lim"])).max() > 1e-3


def test_oracle_feasible_nominal_comes_back_unchanged():
    """A nominal inside the box that keeps every CBF row with margin is its own filtered action, with r = 0."""
    from oracle import qp
    _, _, _, d = _qp_data()
    Lg, b, u_lim = d["Lg_h"], d["b"], d["u_lim"]
    # such a nominal: the QP's solution for rows tightened by 0.05 (then -Lg u <= b - 0.05 without relaxation)
    u_in, r_in, _, _ = qp.solve_qp_dual(Lg, b - 0.05, d["u_ref"], u_lim)
    assert (r_in == 0).all() and (-Lg @ u_in <= b - 0.05 + 1e-9).all() and (np.abs(u_in) <= u_lim).all()
    assert np.abs(u_in - d["u_ref"]).max() > 1e-2                 # not u_ref: a nominal of its own
    u, r, lam, it = qp.solve_qp_dual(Lg, b, u_in, u_lim)
    np.testing.assert_allclose(u, u_in, rtol=0, atol=1e-12)
    assert (r == 0).all() and (lam == 0).all() and it == 1
    kkt = qp.kkt_residual(Lg, b, u_in, u_lim, u, r, lam)
    assert max(kkt.values()) == 0.0, kkt


def test_oracle_nominal_outside_the_box_matches_slsqp():
    """A nominal outside the u_lim box (the policy's 2 pi + u_ref can be): the dual solve agrees with the independent
    primal active-set solve."""
    from oracle import qp
    _, _, _, d = _qp_data()
    Lg, b, u_lim = d["Lg_h"], d["b"], d["u_lim"]
    u_nom = np.random.Generator(np.random.PCG64(5)).uniform(-2 * u_lim, 2 * u_lim, size=Lg.shape[1])
    assert (np.abs(u_nom) > u_lim).any()
    u, r, lam, _ = qp.solve_qp_dual(Lg, b, u_nom, u_lim)
    u2, r2, _ = qp.solve_qp_slsqp(Lg, b, u_nom, u_lim)
    np.testing.assert_allclose(u, u2, atol=1e-6, rtol=0)
    np.testing.assert_allclose(r, r2, atol=1e-6, rtol=0)
    kkt = qp.kkt_residual(Lg, b, u_nom, u_lim, u, r, lam)
    assert max(kkt.values()) < 1e-8, kkt
