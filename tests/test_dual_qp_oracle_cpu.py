"""CPU: the float64 replica of the device QPs' dual ascent (tests/dual_qp_oracle.py) on its own.

* Run to convergence with each caller's knobs, it reaches the minimiser of SciPy's SLSQP on small random problems with
  relaxed rows, an all-zero row and two identical rows, and its (u, r, lam) passes the KKT certificate.
* Its first iteration equals a hand computation on a 2-row problem, with and without the relaxed-row warm start.
* With the labels' knobs an agent whose u_ref is all NaN gets u = -u_lim, and the other agents get the minimiser of
  the QP with that agent's action fixed at -u_lim.
"""
import numpy as np
import pytest

import dual_qp_oracle as dq
from oracle.qp import kkt_residual, solve_qp_slsqp

U_LIM = 1.0


def _problem(seed, identical_rows):
    """6 rows over 4 agents x 2 actions: row 0 relaxed (no u in the box satisfies it), row 1 all zero and relaxed,
    row 3 a copy of row 2 when identical_rows."""
    rng = np.random.Generator(np.random.PCG64(seed))
    M, n = 6, 8
    Lg = rng.normal(size=(M, n))
    Lg[rng.random((M, n)) < 0.4] = 0.0
    b = rng.normal(scale=0.5, size=M)
    u_ref = rng.uniform(-1.5 * U_LIM, 1.5 * U_LIM, size=n)
    b[0] = -np.abs(Lg[0]).sum() * U_LIM - 0.3
    Lg[1] = 0.0
    b[1] = -0.2
    if identical_rows:
        Lg[3], b[3] = Lg[2], b[2]
    return Lg, b, u_ref


@pytest.mark.parametrize("caller", ["labels", "dec_share_cbf", "centralized_cbf"])
@pytest.mark.parametrize("identical_rows", [False, True])
@pytest.mark.parametrize("seed", [1, 2, 4])
def test_converged_replica_is_the_minimiser(caller, identical_rows, seed):
    # draws on which SLSQP itself ends accurate: on some others (seeds 3 and 7) its line search stops with u 1e-3 off,
    # while the replica's KKT residual is 1e-9 on every draw
    Lg, b, u_ref = _problem(seed, identical_rows)
    # the labels keep u in fp32 between iterations: their residual stalls near fp32 rounding, so they stop earlier
    fp32 = caller == "labels"
    run = dq.dual_ascent(Lg, b, u_ref, U_LIM, caller=caller, max_iter=200000, tol=1e-6 if fp32 else 1e-12)
    assert run.converged and run.iters < 200000
    assert run.mu0[0] > 0 and run.mu0[1] > 0, "rows 0 and 1 must start at the relaxed-row warm start"
    us, rs, _ = solve_qp_slsqp(Lg, b, u_ref, U_LIM)
    # two identical rows share their multiplier in any split: lam is not unique, (u, r) is
    np.testing.assert_allclose(run.u, us, atol=1e-4 if fp32 else 1e-6, rtol=0)
    np.testing.assert_allclose(run.r, rs, atol=1e-4 if fp32 else 1e-5, rtol=0)
    np.testing.assert_allclose(run.r[1], 0.2, atol=1e-5)          # the all-zero row: r = max(0, -b)
    kkt = kkt_residual(Lg, b, u_ref, U_LIM, run.u, run.r, run.lam)
    if fp32:
        assert kkt["stationarity_u"] < 1e-6 and kkt["primal"] < 1e-5 and kkt["dual"] == 0.0, kkt
    else:
        assert max(kkt.values()) < 1e-8, kkt
    assert (run.lam > 0).sum() >= 3, "the problem has too few active rows"


@pytest.mark.parametrize("warm", [False, True])
def test_first_iteration_by_hand(warm):
    """Lg = diag(1, 2) over one agent's 2 actions, u_ref = (0.5, -0.25), u_lim = 1.  Row 1 is active from lam = 0;
    with warm, row 0 (b = -1.5) is violated by every u in the box (vmin = 0.5) and starts at lam = 1005, where its
    gradient is exactly 0."""
    Lg = np.array([[1.0, 0.0], [0.0, 2.0]])
    u_ref = np.array([0.5, -0.25])
    b = np.array([-1.5 if warm else 0.2, 0.1])
    s1, s2 = 1 / np.sqrt(1.1), 1 / np.sqrt(4.1)
    lip = max(s1, 2 * s2) ** 2 + max(s1, s2) ** 2 / 10      # |S Lg|_1 |S Lg|_inf + max s^2 / 10
    run = dq.dual_ascent(Lg, b, u_ref, U_LIM, caller="centralized_cbf", max_iter=1, tol=0.0)
    assert run.iters == 1 and not run.converged
    np.testing.assert_allclose(run.lip, lip, rtol=1e-15)
    # iteration 1: grad_1 = s2 (-2 u_1 - b_1) = 0.4 s2, mu_1 = grad_1 / L, no restart (grad . mu_new > 0)
    mu1 = 0.4 * s2 / lip
    np.testing.assert_allclose(run.res_lip, [0.4 * s2], rtol=1e-14)
    if warm:
        np.testing.assert_allclose(run.mu0, [1005 / s1, 0.0], rtol=1e-15)
        np.testing.assert_allclose(run.lam, [1005.0, s2 * mu1], rtol=1e-13)
        np.testing.assert_allclose(run.r, [0.5, 0.0], rtol=0, atol=1e-12)
        np.testing.assert_allclose(run.u, [1.0, -0.25 + 2 * s2 * mu1], rtol=1e-14)
    else:
        np.testing.assert_array_equal(run.mu0, [0.0, 0.0])
        # grad_0 = s1 (-u_0 - b_0) = -0.7 s1 < 0: row 0 stays at 0
        np.testing.assert_allclose(run.lam, [0.0, s2 * mu1], rtol=1e-14)
        np.testing.assert_array_equal(run.r, [0.0, 0.0])
        np.testing.assert_allclose(run.u, [0.5, -0.25 + 2 * s2 * mu1], rtol=1e-14)
    # restart margin |grad . d| / (|grad| |d|), d = mu_new - mu = (0, mu_1)
    grad0 = 0.0 if warm else -0.7 * s1
    assert run.margin[0] == pytest.approx(0.4 * s2 / np.hypot(grad0, 0.4 * s2), rel=1e-12)


def test_labels_nan_u_ref_clips_to_minus_u_lim():
    rng = np.random.Generator(np.random.PCG64(7))
    N, nu = 4, 2
    Lg = rng.normal(size=(N, N * nu))
    b = rng.normal(scale=0.3, size=N)
    u_ref = rng.uniform(-0.8, 0.8, size=N * nu)
    u_ref[:nu] = np.nan                                       # agent 0 sits exactly at its goal
    run = dq.dual_ascent(Lg, b, u_ref, U_LIM, caller="labels", max_iter=200000, tol=1e-6)
    assert run.converged
    np.testing.assert_array_equal(run.u[:nu], -U_LIM)
    assert np.isfinite(run.u).all() and np.isfinite(run.lam).all()
    # the other agents: the QP with agent 0's action fixed at -u_lim (its columns moved into b)
    b_fix = b + Lg[:, :nu] @ np.full(nu, -U_LIM)
    us, rs, _ = solve_qp_slsqp(Lg[:, nu:], b_fix, u_ref[nu:], U_LIM)
    np.testing.assert_allclose(run.u[nu:], us, atol=1e-4, rtol=0)
    np.testing.assert_allclose(run.r, rs, atol=1e-4, rtol=0)
    assert (run.lam > 0).any(), "no row active: agent 0's fixed action would not matter"
    # the baselines' rule on the same data: 0 in the ascent, NaN in the result
    base = dq.dual_ascent(Lg, b, u_ref, U_LIM, caller="centralized_cbf", max_iter=200000, tol=1e-12)
    assert np.isnan(base.u[:nu]).all() and np.isfinite(base.u[nu:]).all()
