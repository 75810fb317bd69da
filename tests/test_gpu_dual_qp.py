"""GPU: the dual ascent of every device QP (csrc/dual_qp.cuh) -- the GCBF+ labels, the safety filter, DecShareCBF and
CentralizedCBF -- against the float64 replica of its schedule (tests/dual_qp_oracle.py), and the solvers at the sizes
where their kernels stride, fall back or fill shared memory.

* Iterate parity: with tol = 0 and max_iter = k, each caller returns the replica's iterate at k (u, and lam or r) and
  reports k (the baselines with the cap bit set).  A wrong momentum, restart, warm start or returned iterate still
  converges to the same minimiser; it does not give the same iterate.  The replica runs on the device's own data:
  the assembled workspace (labels, filter; s from QSC) and the pairwise blocks (baselines; b formed as the kernels form
  it).  The remaining gap is the step bound computed in fp32 and the fma and sum order.  A case whose restart decision
  is within rounding (the replica's margin |grad . d| / (|grad| |d|) < 1e-6 at some iteration up to k) is skipped
  and counted.
* Stop rule: with tol just above the replica's res L at an iteration k that is a new minimum by 1 %, the device stops
  at exactly k with the replica's iterate; with tol just below it and max_iter = k it reports k as a capped solve.
* Sizes: the labels and the filter at N = 1025 (1024 threads, two rows on thread 0) and N = 2048 on both neighbour
  paths, CentralizedCBF at its limits (DoubleIntegrator 1024, LinearDrone 999), each against the float64 minimiser of
  its own data and the KKT certificate of tests/test_gpu_qp.py, with no capped solve.
* Edges with known answers: a pairwise row with Lg = 0 (two coincident agents), and the labels' NaN u_ref rule.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import cbfqp_oracle as cq
import dual_qp_oracle as dq
from helpers import product_algo, product_env, product_obstacles, random_scene
from oracle import qp
from test_gpu_qp import _qp_from_device

pytestmark = pytest.mark.gpu

FLAG = 1 << 30
KS = (1, 2, 5, 25)
MARGIN = 1e-6
CALLERS = ("labels", "filter", "dec_share_cbf", "centralized_cbf")


# ------------------------------------------------------------------------------------------------------ scenes
def _pd(env_id):
    return 3 if env_id == "LinearDrone" else 2


def _labels_scene(env_id, N, G, area, n_obs, seed, vs=4.0, gap=0.05, pairs=(0, 2, 4)):
    """Random states plus head-on pairs (agent a and a + 1, `gap` apart, closing at 2 vs): the learned CBF then has rows
    that no action in the box satisfies (relaxed rows, where the warm start runs)."""
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=seed)
    pd = _pd(env_id)
    e = np.ones(pd, np.float32) / np.sqrt(pd)
    for a in pairs:
        agent[:, a + 1, :pd] = agent[:, a, :pd] + gap * e
        agent[:, a, pd:2 * pd] = vs * e
        agent[:, a + 1, pd:2 * pd] = -vs * e
    return _build(env_id, N, area, n_obs, agent, goal, obs)


def _build(env_id, N, area, n_obs, agent, goal, obs, edge_cap=64):
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = edge_cap
    algo = product_algo(env, env_id)
    pobs = product_obstacles(env_id, obs) if n_obs else None
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    return env, algo, graph


def _baseline_scene(env_id, N, G, seed, gap):
    """Random states without obstacles plus a co-moving pair `gap` apart in every graph: its two pairwise rows have
    h < 0, Lf_h = 0 and a tiny Lg (relaxed rows)."""
    area = 1.5 if env_id == "DoubleIntegrator" else 0.8
    agent, goal, _ = random_scene(env_id, N, G, area, 0, seed=seed)
    pd = _pd(env_id)
    agent[:, 1, :pd] = agent[:, 0, :pd] + gap / np.sqrt(pd)
    agent[:, 1, pd:] = agent[:, 0, pd:]
    env = product_env(env_id, N, area, 0)
    return env, env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), None)


# ------------------------------------------------------------------------------------------------------ device calls
def _abi_qp(env, algo, graph, u_nom, max_iter, tol):
    """gcbf_qp_labels (u_nom None) or gcbf_qp_filter on a fresh workspace: (u, aux, raw iteration words, workspace)."""
    from gcbfplus_b200 import _lib
    G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
    d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
    ws = torch.empty(int(env.lib.gcbf_qp_workspace_floats(C.byref(d))), dtype=torch.float32, device="cuda")
    u = torch.empty(G, N, nu, dtype=torch.float32, device="cuda")
    aux = torch.empty(G, N, 2, dtype=torch.float32, device="cuda")
    iters = torch.empty(G, dtype=torch.int32, device="cuda")
    head = (C.byref(d), float(algo.alpha), 1 if _lib.USE_TC else 0, int(max_iter), float(tol),
            _lib.ptr(algo.cbf_params.flat), _lib.ptr(graph.agent), _lib.ptr(graph.goal), _lib.ptr(graph.hits),
            _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_recv), _lib.ptr(graph.edge_src),
            _lib.ptr(graph.counters))
    tail = (_lib.ptr(u), _lib.ptr(aux), _lib.ptr(iters), _lib.ptr(ws), ws.numel(), env._stream())
    if u_nom is None:
        _lib.check(env.lib.gcbf_qp_labels(*head, *tail), "gcbf_qp_labels")
    else:
        _lib.check(env.lib.gcbf_qp_filter(*head, _lib.ptr(u_nom), *tail), "gcbf_qp_filter")
    torch.cuda.synchronize()
    graph.check_overflow()
    return u.cpu().numpy().astype(np.float64), aux.cpu().numpy().astype(np.float64), iters.cpu().numpy(), ws


def _controller(env, name, **kw):
    from gcbfplus_b200.algo import make_algo
    return make_algo(name, env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=env.num_agents, **kw)


def _baseline(env, graph, name, max_iter, tol):
    ctl = _controller(env, name, max_iter=max_iter, tol=tol)
    u, r = ctl.get_qp_action(graph)
    torch.cuda.synchronize()
    return (u.cpu().numpy().astype(np.float64), r.cpu().numpy().astype(np.float64),
            ctl.last_iters.cpu().numpy().reshape(graph.n_graphs, -1))


# ------------------------------------------------------------------------------------------------------ problems
class Problem:
    """One QP of a caller on the device's own data, and the device's answer for it: `solve(max_iter, tol)` runs the
    device and returns for this problem (u [n], lam or r [M], raw iteration word)."""

    def __init__(self, caller, Lg, b, u_ref, u_lim, s, solve, lam_out):
        self.caller, self.Lg, self.b, self.u_ref, self.u_lim, self.s = caller, Lg, b, u_ref, u_lim, s
        self.solve, self.lam_out = solve, lam_out      # lam_out: the device returns lam (labels) or r (baselines)

    def replica(self, max_iter, tol):
        return dq.dual_ascent(self.Lg, self.b, self.u_ref, self.u_lim, self.s, caller=self.caller, max_iter=max_iter,
                              tol=tol)

    def n_relaxed(self):
        return int((dq.warm_start(self.Lg, self.b, self.s, self.u_lim) > 0).sum())


def _qp_problems(env, algo, graph, u_nom):
    """Labels (u_nom None) or filter problems, one per graph."""
    N, nu = env.num_agents, env.action_dim
    u_lim = float(env.action_lim()[1][0])
    un = None if u_nom is None else torch.from_numpy(u_nom).cuda()
    _, _, _, ws = _abi_qp(env, algo, graph, un, 1, 0.0)
    data = _qp_from_device(env, ws, graph, N, nu, sparse=True)
    caller = "labels" if u_nom is None else "filter"
    memo = {}

    def run(max_iter, tol):
        if (max_iter, tol) not in memo:
            memo[(max_iter, tol)] = _abi_qp(env, algo, graph, un, max_iter, tol)[:3]
        return memo[(max_iter, tol)]

    def solver(g):
        def solve(max_iter, tol):
            u, aux, it = run(max_iter, tol)
            return u[g].reshape(-1), aux[g, :, 0], int(it[g])
        return solve
    return [Problem(caller, d["Lg"], d["b"], d["u_ref"], u_lim, d["s"], solver(g), True) for g, d in enumerate(data)]


def _pairwise_np(env, graph):
    p = _controller(env, "dec_share_cbf").pairwise(graph)
    return {k: v.cpu().numpy() for k, v in p.items()}


def _baseline_problems(env, graph, name):
    """DecShareCBF: one problem per agent (b = fp32 resp (lf + alpha h)); CentralizedCBF: one per graph
    (b = lf + alpha h), s as the kernels form it from the fp32 blocks."""
    G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
    u_lim = float(env.action_lim()[1][0])
    p = _pairwise_np(env, graph)
    u_ref = env.u_ref(graph).cpu().numpy().astype(np.float64)
    one = np.float32(1.0)
    memo = {}

    def run(max_iter, tol):
        if (max_iter, tol) not in memo:
            memo[(max_iter, tol)] = _baseline(env, graph, name, max_iter, tol)
        return memo[(max_iter, tol)]

    out = []
    for g in range(G):
        lf, h, ls = p["lf_h"][g], p["h"][g], p["lg_self"][g]
        if name == "dec_share_cbf":
            resp = np.where(p["isobs"][g], np.float32(1.0), np.float32(0.5))
            b = (resp * (lf + one * h)).astype(np.float64)
            for i in range(N):
                Lg = ls[i].astype(np.float64)
                s = 1.0 / np.sqrt((Lg * Lg).sum(1) + 0.1)

                def solve(max_iter, tol, g=g, i=i):
                    u, r, it = run(max_iter, tol)
                    return u[g, i], r[g, i], int(it[g, i])
                out.append(Problem(name, Lg, b[i], u_ref[g, i], u_lim, s, solve, False))
        else:
            Lg = cq.central_from_blocks(p["idx"][g], ls, p["lg_other"][g])
            b = (lf + one * h).astype(np.float64).reshape(-1)
            sq = (ls * ls + p["lg_other"][g] * p["lg_other"][g]).sum(-1, dtype=np.float32).reshape(-1)
            s = (1.0 / np.sqrt(sq.astype(np.float64) + np.float32(0.1))).astype(np.float32).astype(np.float64)

            def solve(max_iter, tol, g=g):
                u, r, it = run(max_iter, tol)
                return u[g].reshape(-1), r[g].reshape(-1), int(it[g, 0])
            out.append(Problem(name, Lg, b, u_ref[g].reshape(-1), u_lim, s, solve, False))
    return out


def _parity_problems(caller, env_id):
    if caller in ("labels", "filter"):
        N, G, area, n_obs, seed = (16, 3, 1.6, 8, 1) if env_id == "DoubleIntegrator" else (10, 2, 1.0, 4, 6)
        env, algo, graph = _labels_scene(env_id, N, G, area, n_obs, seed)
        u_nom = None
        if caller == "filter":
            u_lim = float(env.action_lim()[1][0])
            rng = np.random.Generator(np.random.PCG64(seed + 100))
            u_nom = rng.uniform(-2 * u_lim, 2 * u_lim, size=(G, N, env.action_dim)).astype(np.float32)
            assert (np.abs(u_nom) > u_lim).any()
        return _qp_problems(env, algo, graph, u_nom)
    gap = 5e-4 if env_id == "DoubleIntegrator" else 1e-4
    env, graph = _baseline_scene(env_id, 16, 3, seed=5, gap=gap)
    return _baseline_problems(env, graph, caller)


# ------------------------------------------------------------------------------------------------------ checks
def _iterate_err(got, want, rel, atol):
    """Largest |got - want| / (rel |want| + atol) (<= 1 passes)."""
    return float((np.abs(got - want) / (rel * np.abs(want) + atol)).max())


def _check_iterate(pb, got_u, got_l, run, what):
    want_l = run.lam if pb.lam_out else run.r
    # lam ~ 1e3 on a relaxed row is exported in fp32; r = (lam - 1000) / 10 inherits lam's absolute error
    scale = max(1.0, float(np.abs(run.lam).max()))
    eu = _iterate_err(got_u, run.u, 1e-4, 1e-6)
    el = _iterate_err(got_l, want_l, 1e-4, 1e-6 * scale)
    assert eu <= 1 and el <= 1, (what, eu, el, np.abs(got_u - run.u).max(), np.abs(got_l - want_l).max())
    return max(eu, el)


@pytest.mark.parametrize("env_id", ["DoubleIntegrator", "LinearDrone"])
@pytest.mark.parametrize("caller", CALLERS)
def test_iterate_parity_at_fixed_count(caller, env_id):
    probs = _parity_problems(caller, env_id)
    relaxed = [pb.n_relaxed() for pb in probs]
    # the learned LinearDrone CBF gives no relaxed row in the head-on scenes (its |Lg|_1 u_lim outweighs b): its
    # labels and filter check the warm start through the DoubleIntegrator scenes only
    if not (caller in ("labels", "filter") and env_id == "LinearDrone"):
        assert sum(relaxed) > 0, f"{caller} {env_id}: no relaxed row, the warm start would not run"
    compared, skipped, worst = 0, 0, 0.0
    ks_compared = set()
    for k in KS:
        n_cmp = n_skip = 0
        for j, pb in enumerate(probs):
            run = pb.replica(k, 0.0)
            if run.margin.min() < MARGIN:
                n_skip += 1
                continue
            u, l, it = pb.solve(k, 0.0)
            flag = FLAG if caller in ("dec_share_cbf", "centralized_cbf") else 0
            assert it == k | flag, (caller, k, j, hex(it))
            worst = max(worst, _check_iterate(pb, u, l, run, (caller, env_id, k, j)))
            n_cmp += 1
        compared += n_cmp
        skipped += n_skip
        # a k counts as compared when (nearly) every problem was
        if n_cmp >= 0.9 * len(probs):
            ks_compared.add(k)
    print(f"{caller} {env_id}: {len(probs)} problems, relaxed rows {sum(relaxed)} (per problem max {max(relaxed)}); "
          f"k-parity compared {compared}, skipped {skipped}, k compared {sorted(ks_compared)}, worst err/tol {worst:.3g}")
    assert len(ks_compared) >= 3, ks_compared


def _stop_k(run, lo=3):
    """An iteration k >= lo whose res L is a new minimum by at least 1 % and whose restarts up to k are not within
    rounding."""
    rl = run.res_lip
    for k in range(lo, len(rl) + 1):
        if run.margin[:k].min() < MARGIN:
            return None
        if rl[k - 1] > 0 and rl[k - 1] < 0.99 * rl[:k - 1].min():
            return k
    return None


@pytest.mark.parametrize("caller", CALLERS)
def test_stop_rule(caller):
    probs = _parity_problems(caller, "DoubleIntegrator")
    capped_flag = FLAG if caller in ("dec_share_cbf", "centralized_cbf") else 0
    # the problem with the most active rows whose sequence has a qualifying k
    order = sorted(range(len(probs)), key=lambda j: -int((probs[j].replica(200, 1e-30).lam > 0).sum()))
    for j in order:
        pb = probs[j]
        full = pb.replica(200, 0.0)
        k = _stop_k(full)
        if k is not None and (full.lam > 0).any():
            break
    else:
        pytest.fail(f"{caller}: no problem has a qualifying stop iteration")
    rk = float(full.res_lip[k - 1])
    at_k = pb.replica(k, 0.0)
    tol = float(np.float32(1.005 * rk))
    run = pb.replica(k + 200, tol)
    assert run.converged and run.iters == k
    u, l, it = pb.solve(k + 200, tol)
    assert it == k, (caller, k, hex(it))
    _check_iterate(pb, u, l, at_k, (caller, "stop", k))
    tol = float(np.float32(0.995 * rk))
    u, l, it = pb.solve(k, tol)
    assert it == k | capped_flag, (caller, k, hex(it))
    _check_iterate(pb, u, l, at_k, (caller, "cap", k))
    print(f"{caller}: stop rule at k = {k} (res L {rk:.4g}) on problem {j}")


# ------------------------------------------------------------------------------------------------------ sizes
def _kkt_ok(Lg, b, u_ref, u_lim, u, r, lam):
    kkt = qp.kkt_residual(Lg, b, u_ref, u_lim, u, r, lam)
    assert kkt["stationarity_u"] < 1e-4 and kkt["primal"] < 1e-3 and kkt["dual"] == 0.0, kkt


def _labels_at_size(env_id, N, area, n_obs, seed, max_iter=60000, tol=1e-6):
    """Labels and filter on one graph of N agents, each against the float64 minimiser of its own data; returns the
    iteration words [labels, filter]."""
    agent, goal, obs = random_scene(env_id, N, 1, area, n_obs, seed=seed)
    env, algo, graph = _build(env_id, N, area, n_obs, agent, goal, obs)
    u_lim = float(env.action_lim()[1][0])
    rng = np.random.Generator(np.random.PCG64(seed))
    u_nom = rng.uniform(-2 * u_lim, 2 * u_lim, size=(1, N, env.action_dim)).astype(np.float32)
    words = []
    for un in (None, torch.from_numpy(u_nom).cuda()):
        u, aux, it, ws = _abi_qp(env, algo, graph, un, max_iter, tol)
        d = _qp_from_device(env, ws, graph, N, env.action_dim, sparse=True)[0]
        n_it = int(it[0]) & (FLAG - 1)
        assert n_it < max_iter, "capped"
        uo, ro, lam, _ = cq.solve_dual_batched(d["Lg"], d["b"], d["u_ref"], u_lim)
        ud = u[0].reshape(-1)
        np.testing.assert_allclose(ud, uo, atol=2e-4, rtol=0)
        np.testing.assert_allclose(aux[0, :, 0], lam, atol=1e-3, rtol=1e-3)
        np.testing.assert_allclose(aux[0, :, 1], ro, atol=1e-3, rtol=1e-3)
        _kkt_ok(d["Lg"], d["b"], d["u_ref"], u_lim, ud, aux[0, :, 1], aux[0, :, 0])
        assert (lam > 0).sum() > 0, "no active row"
        words.append(int(it[0]))
        print(f"{env_id} N={N} {'labels' if un is None else 'filter'}: {n_it} iterations, "
              f"{'global' if it[0] & FLAG else 'shared'} path, {int((lam > 0).sum())} active rows, "
              f"{int(graph.row_deg.sum())} edges")
    return words


def test_labels_and_filter_at_1025_agents():
    """1025 agents: 1024 threads, thread 0 owns rows 0 and 1024."""
    _labels_at_size("DoubleIntegrator", 1025, 10.0, 8, seed=31)


@pytest.mark.parametrize("env_id", ["DoubleIntegrator", "LinearDrone"])
@pytest.mark.parametrize("density", ["sparse", "normal"])
def test_labels_and_filter_at_2048_agents(env_id, density):
    """2048 agents: the shared-memory neighbour budget is set by the 200 KB cap (about 2 blocks per agent for NU = 2,
    1 for NU = 3).  A sparse scene keeps its blocks in shared memory; a normal-density one takes the global path."""
    area = {("DoubleIntegrator", "sparse"): 57.0, ("DoubleIntegrator", "normal"): 24.0,
            ("LinearDrone", "sparse"): 15.0, ("LinearDrone", "normal"): 6.5}[(env_id, density)]
    words = _labels_at_size(env_id, 2048, area, 8 if env_id == "DoubleIntegrator" else 4, seed=32)
    for w in words:
        assert bool(w & FLAG) == (density == "normal"), (env_id, density, hex(w))


@pytest.mark.parametrize("env_id,N", [("DoubleIntegrator", 1024), ("LinearDrone", 999)])
def test_centralized_at_its_limits(env_id, N):
    """DoubleIntegrator 1024 agents (3072 rows, 6 per thread); LinearDrone 999 (164 B under the 227 KB opt-in)."""
    from test_gpu_cbfqp import _graph
    env, g, _, _ = _graph(env_id, N, 1, seed=40)
    u, r, it = _baseline(env, g, "centralized_cbf", 200000, 1e-8)
    assert not (it & FLAG).any(), "capped"
    pb = _baseline_problems(env, g, "centralized_cbf")[0]
    uo, ro, lam, _ = cq.solve_dual_batched(pb.Lg, pb.b, pb.u_ref, pb.u_lim)
    np.testing.assert_allclose(u[0].reshape(-1), uo, atol=1e-5)
    np.testing.assert_allclose(r[0].reshape(-1), ro, atol=1e-4)
    # the baselines export no multipliers: the certificate takes the exact ones
    _kkt_ok(pb.Lg, pb.b, pb.u_ref, pb.u_lim, u[0].reshape(-1), r[0].reshape(-1), lam)
    assert (lam > 1e-9).sum() > 0
    print(f"centralized_cbf {env_id} N={N}: {int(it[0, 0])} iterations, {int((lam > 1e-9).sum())} active rows")


# ------------------------------------------------------------------------------------------------------ edges
def test_zero_row_from_coincident_agents():
    """Two coincident SingleIntegrator agents: their pairwise row has Lg = 0 and h = -4 (1.01 r)^2, so r = max(0, -b).
    The warm start lands on the optimum; every other row is inactive, so the solve stops after 1 iteration."""
    agent = np.array([[[1.0, 1.0], [1.0, 1.0], [3.0, 1.0], [1.0, 3.0]]], np.float32)
    goal = agent.copy()
    goal[..., 0] += 0.01
    env = product_env("SingleIntegrator", 4, 4.0, 0)
    g = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), None)
    p = _pairwise_np(env, g)
    assert (p["idx"][0, :2, 0] == [1, 0]).all()
    assert (p["lg_self"][0, :2, 0] == 0).all() and (p["lg_other"][0, :2, 0] == 0).all() and (p["lf_h"][0, :2, 0] == 0).all()
    for name in ("dec_share_cbf", "centralized_cbf"):
        u, r, it = _baseline(env, g, name, 10000, 1e-8)
        assert np.isfinite(u).all() and np.isfinite(r).all(), name
        resp = np.float32(0.5) if name == "dec_share_cbf" else np.float32(1.0)
        b = resp * (p["lf_h"][0, :2, 0] + np.float32(1.0) * p["h"][0, :2, 0])
        np.testing.assert_allclose(r[0, :2, 0], np.maximum(0, -b.astype(np.float64)), rtol=2e-7, atol=0)
        assert (r[0, :, 1:] == 0).all() and (r[0, 2:] == 0).all(), name
        assert (it == 1).all(), (name, it)


def test_labels_nan_u_ref_at_goal():
    """A DoubleIntegrator agent exactly at its goal has a NaN u_ref: the labels clip it to -u_lim.  Every other agent
    gets the float64 minimiser of the QP with that agent's action fixed at -u_lim (u_ref = -inf)."""
    env_id, N, G, area, n_obs = "DoubleIntegrator", 8, 2, 1.5, 4
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=11)
    agent[0, 3] = goal[0, 3]
    env, algo, graph = _build(env_id, N, area, n_obs, agent, goal, obs)
    u, aux, it, ws = _abi_qp(env, algo, graph, None, 20000, 1e-6)
    data = _qp_from_device(env, ws, graph, N, env.action_dim, sparse=True)
    u_lim = float(env.action_lim()[1][0])
    nan_ref = np.isnan(data[0]["u_ref"])
    assert nan_ref.sum() == env.action_dim and nan_ref.reshape(N, -1)[3].all()
    assert (u[0, 3] == -np.float32(u_lim)).all()
    assert np.isfinite(u).all() and np.isfinite(aux).all()
    for gi, d in enumerate(data):
        ur = np.where(np.isnan(d["u_ref"]), -np.inf, d["u_ref"])
        uo, ro, lam, _ = cq.solve_dual_batched(d["Lg"], d["b"], ur, u_lim)
        np.testing.assert_allclose(u[gi].reshape(-1), uo, atol=2e-4, rtol=0)
        np.testing.assert_allclose(aux[gi, :, 0], lam, atol=1e-3, rtol=1e-3)
        assert int(it[gi]) & (FLAG - 1) < 20000
