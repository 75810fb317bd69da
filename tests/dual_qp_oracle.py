"""Float64 replica of the device QPs' dual ascent (csrc/dual_qp.cuh), iterate by iterate (TEST INFRASTRUCTURE ONLY --
never imported by the product).

`oracle.qp.solve_qp_dual` and `cbfqp_oracle.solve_dual_batched` give the QP's unique minimiser; a solver that reaches
it by another schedule (a wrong momentum, restart, warm start or returned iterate) passes every test built on them.
This module runs the device schedule exactly, so that a test can stop the device after k iterations and compare
iterates:

    mu = y = warm start ((1000 + 10 vmin) / s where vmin = -|Lg_i|_1 u_lim - b_i > 0, else 0), t = 1
    each iteration:  lam = s y,  u = u(lam),  grad = s (-Lg u - r(lam) - b),  mu_new = max(0, y + grad / L)
                     res = max |mu_new - y|,  restart when grad . (mu_new - mu) < 0 (t = 1, beta = 0),
                     else t_new = (1 + sqrt(1 + 4 t^2)) / 2, beta = (t - 1) / t_new
                     y = mu_new + beta (mu_new - mu),  mu = mu_new,  stop when res L < tol (after the update)
    returned iterate: lam = s mu, u = u(lam), r = r(lam); the count is min(it, max_iter)

The callers' own choices are knobs, named as DESIGN §4.4 names them (`CALLERS`): the step bound L, the precision of
the momentum scalar t and of the primal u kept between iterations, and the NaN u_ref rule.  Everything else is
float64.  The problem is one QP in sparse form: Lg [M, n] (scipy CSR), b [M], u_ref [n], u_lim and the row scale s [M].
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import scipy.sparse as sp

from oracle.qp import RELAX_PENALTY, RELAX_WEIGHT

#: per-caller knobs: step bound, momentum t dtype, primal u dtype, NaN u_ref rule
CALLERS = {
    # L = |S Lg|_1 |S Lg|_inf + max(s^2) / 10; t and u in fp32; a NaN u_ref component clips to -u_lim
    "labels": dict(step_bound="norm1_norminf", momentum=np.float32, primal=np.float32, nan_u_ref="clip"),
    # L = |S Lg|_F^2 + max(s^2) / 10; fp64; a NaN u_ref component is 0 in the ascent and NaN in the result
    "dec_share_cbf": dict(step_bound="frobenius", momentum=np.float64, primal=np.float64, nan_u_ref="zero"),
    "centralized_cbf": dict(step_bound="norm1_norminf", momentum=np.float64, primal=np.float64, nan_u_ref="zero"),
}
CALLERS["filter"] = CALLERS["labels"]


def row_scale(Lg) -> np.ndarray:
    """s = 1 / sqrt(|row|^2 + 0.1)."""
    Lg = sp.csr_matrix(Lg, dtype=np.float64)
    return 1.0 / np.sqrt(np.asarray(Lg.multiply(Lg).sum(1)).ravel() + 1.0 / RELAX_WEIGHT)


def step_bound(Lg, s: np.ndarray, kind: str) -> float:
    """L = norm + max(s^2) / 10 with norm >= |S Lg|_2^2 ("norm1_norminf": |S Lg|_1 |S Lg|_inf, "frobenius":
    |S Lg|_F^2)."""
    A = abs(sp.diags(s) @ sp.csr_matrix(Lg, dtype=np.float64))
    if kind == "norm1_norminf":
        norm = float(np.asarray(A.sum(0)).max()) * float(np.asarray(A.sum(1)).max())
    elif kind == "frobenius":
        norm = float(A.multiply(A).sum())
    else:
        raise ValueError(kind)
    return norm + float((s * s).max()) / RELAX_WEIGHT


def warm_start(Lg, b: np.ndarray, s: np.ndarray, u_lim: float) -> np.ndarray:
    """mu0: (1000 + 10 vmin) / s on a row no u in the box satisfies (vmin = -|Lg_i|_1 u_lim - b_i > 0), else 0."""
    vmin = -np.asarray(abs(sp.csr_matrix(Lg, dtype=np.float64)).sum(1)).ravel() * u_lim - b
    return np.where(vmin > 0, (RELAX_PENALTY + RELAX_WEIGHT * vmin) / s, 0.0)


def relax(lam: np.ndarray) -> np.ndarray:
    return np.maximum(0.0, (lam - RELAX_PENALTY) / RELAX_WEIGHT)


@dataclass
class DualRun:
    u: np.ndarray            # [n] the returned iterate's primal (NaN where the caller's rule returns NaN)
    r: np.ndarray            # [M]
    lam: np.ndarray          # [M]  s mu
    iters: int               # min(it, max_iter)
    converged: bool          # the stop test passed
    res_lip: np.ndarray      # [iters] res * L of each iteration
    margin: np.ndarray       # [iters] |grad . d| / (|grad| |d|), d = mu_new - mu (inf where |grad| |d| = 0)
    lip: float
    mu0: np.ndarray          # [M] the warm start


def dual_ascent(Lg, b, u_ref, u_lim: float, s=None, *, caller: str = "centralized_cbf", max_iter: int,
                tol: float, lip: float | None = None) -> DualRun:
    """Run the device schedule for at most max_iter iterations (tol = 0: exactly max_iter).  s defaults to
    `row_scale(Lg)`, lip to `step_bound(Lg, s, <the caller's bound>)`."""
    k = CALLERS[caller]
    Lg = sp.csr_matrix(Lg, dtype=np.float64)
    LgT = Lg.T.tocsr()
    b = np.asarray(b, np.float64)
    u_ref = np.asarray(u_ref, np.float64)
    s = row_scale(Lg) if s is None else np.asarray(s, np.float64)
    lip = step_bound(Lg, s, k["step_bound"]) if lip is None else float(lip)
    step = 1.0 / lip
    nan_ref = np.isnan(u_ref)
    if k["nan_u_ref"] == "clip":
        u_ref = np.where(nan_ref, -np.inf, u_ref)       # fmax(NaN, -u_lim) = -u_lim
    P, T = k["primal"], k["momentum"]

    def primal(lam, last):
        u = np.clip(u_ref + LgT @ lam, -u_lim, u_lim)
        if k["nan_u_ref"] == "zero":
            u = np.where(nan_ref, np.nan if last else 0.0, u)
        return u.astype(P).astype(np.float64)

    mu0 = warm_start(Lg, b, s, u_lim)
    mu, y = mu0.copy(), mu0.copy()
    t = T(1)
    res_lip, margin = [], []
    conv = False
    it = 0
    for it in range(1, max_iter + 1):
        lam = s * y
        u = primal(lam, False)
        grad = s * (-(Lg @ u) - relax(lam) - b)
        mn = np.maximum(0.0, y + step * grad)
        res = float(np.abs(mn - y).max()) if mn.size else 0.0
        d = mn - mu
        dotp = float(grad @ d)
        den = float(np.linalg.norm(grad) * np.linalg.norm(d))
        margin.append(abs(dotp) / den if den > 0 else np.inf)
        if dotp < 0.0:
            t, beta = T(1), 0.0
        else:
            t_new = T(0.5) * (T(1) + np.sqrt(T(1) + T(4) * t * t))
            beta = float((t - T(1)) / t_new)
            t = t_new
        y = mn + beta * d
        mu = mn
        res_lip.append(res * lip)
        if res * lip < tol:
            conv = True
            break
    lam = s * mu
    return DualRun(u=primal(lam, True), r=relax(lam), lam=lam, iters=min(it, max_iter), converged=conv,
                   res_lip=np.asarray(res_lip), margin=np.asarray(margin), lip=lip, mu0=mu0)
