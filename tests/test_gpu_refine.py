"""GPU parity: online policy refinement (gcbf_refine_actions, GCBFPlus.online_policy_refinement, the rollout engine's
actor_refine policy) vs the oracle's torch-autograd restatement of gcbf.py:161-201 (tests/refine_oracle.py), on both
GEMM paths, all four environments, pretrained and randomly initialised networks.

Tolerances.  One iteration against float64: the loop value 2e-4 + 1e-3 relative (h is divided by dt = 0.03, so fp32
rounding of h ~ 1e-6 reaches the value at ~3e-5), the refined action 1e-4; xavier networks must meet them outright,
pretrained ones may instead stay inside the float64 oracle's own ReLU-kink envelope (as tests/test_gpu_train.py).  The
full loop against the float32 oracle: actions 2e-3 (up to 30 gradient steps, each through an independently rounded
backward) and identical iteration counts, except on graphs whose float64 loop value at the deciding iteration, or one of
whose selection terms, lies within 1e-3 of 0 (those may legitimately decide the other way in fp32); such graphs are
counted and must stay a small minority."""
import argparse
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

from helpers import (ROOT, oracle_env, oracle_obstacles, product_algo, product_env, product_obstacles, random_scene)
from refine_oracle import refine_oracle

pytestmark = pytest.mark.gpu

CASES = [("SingleIntegrator", 8, 3, 0.9, 4, 3), ("DoubleIntegrator", 12, 3, 1.2, 6, 1),
         ("DubinsCar", 10, 3, 1.2, 6, 5), ("LinearDrone", 8, 3, 0.8, 4, 6)]
MARGIN = 1e-3
KINK_DELTA = 1e-4


class _ShiftedReLU(torch.autograd.Function):
    """relu(x) whose derivative is taken as 1[x > delta]: the forward value is the ordinary ReLU
    (copied from tests/test_gpu_train.py)."""

    @staticmethod
    def forward(ctx, x, delta):
        ctx.save_for_backward(x)
        ctx.delta = delta
        return x.clamp_min(0)

    @staticmethod
    def backward(ctx, g):
        (x,) = ctx.saved_tensors
        return g * ((x > ctx.delta) & (x != 0)).to(g.dtype), None


class shifted_relu_derivative:
    """Context manager: every torch.relu of the oracle differentiates as 1[x > delta] (forward unchanged)."""

    def __init__(self, delta):
        self.delta = delta

    def __enter__(self):
        self._orig = torch.relu
        torch.relu = lambda x: _ShiftedReLU.apply(x, self.delta)

    def __exit__(self, *exc):
        torch.relu = self._orig
        return False


def _setup(env_id, N, G, area, n_obs, seed, pretrained, vel_scale=0.45):
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed, vel_scale=vel_scale)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 64
    algo = product_algo(env, env_id if pretrained else None, seed=3)
    pobs = product_obstacles(env_id, obs)
    return env, algo, agent, goal, pobs


def _graph(env, agent, goal, pobs):
    return env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)


def _oracle_setup(env_id, N, area, n_obs, algo, agent, goal, packed, dt):
    from oracle.nn import to_torch
    oenv = oracle_env(env_id, N, area, n_obs, dtype=dt)
    cp = to_torch(algo.cbf_params.to_tree(), dt)
    ap = to_torch(algo.actor_net_params.to_tree(), dt)
    graphs = [oenv.sparsify(oenv.get_graph(torch.from_numpy(agent[g]).to(dt), torch.from_numpy(goal[g]).to(dt),
                                           oracle_obstacles(packed[g], dt))) for g in range(agent.shape[0])]
    return oenv, cp, ap, graphs


def _refine(algo, graph, **kw):
    a, v, it = algo.online_policy_refinement(graph, return_info=True, **kw)
    torch.cuda.synchronize()
    graph.check_overflow()
    return a.cpu().double(), v.cpu().double(), it.cpu()


@pytest.mark.parametrize("env_id,N,G,area,n_obs,seed", CASES)
@pytest.mark.parametrize("pretrained", [True, False])
def test_one_iteration_matches_float64(env_id, N, G, area, n_obs, seed, pretrained, gemm_path):
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, seed, pretrained)
    graph = _graph(env, agent, goal, pobs)
    a0, _, _ = _refine(algo, graph, lr=0.0, max_iter=1)           # lr = 0: the per-agent selection itself
    a1, v1, it1 = _refine(algo, graph, max_iter=1)
    assert (it1 & 0x3FFFFFFF).eq(1).all()
    oenv, cp, ap, graphs = _oracle_setup(env_id, N, area, n_obs, algo, agent, goal, pobs.packed.cpu().numpy(),
                                         torch.float64)
    n_sel = n_kink = 0
    for g in range(G):
        o0 = refine_oracle(oenv, cp, ap, graphs[g], alpha=algo.alpha, lr=0.0, max_iter=1)
        firm = (o0["sel_term"].abs() > MARGIN).numpy()
        n_sel += int(o0["sel"].sum())
        np.testing.assert_allclose(a0[g].numpy()[firm], o0["action"].numpy()[firm], atol=1e-4, rtol=0)
        o1 = refine_oracle(oenv, cp, ap, graphs[g], alpha=algo.alpha, max_iter=1)
        want_v = o1["values"][0]
        assert abs(float(v1[g]) - want_v) <= 2e-4 + 1e-3 * abs(want_v), (g, float(v1[g]), want_v)
        if not firm.all():
            continue
        err = (a1[g] - o1["action"]).abs()
        if float(err.max()) <= 1e-4:
            continue
        assert pretrained, (g, float(err.max()), "a randomly initialised network has no ReLU ties: strict tolerance")
        with shifted_relu_derivative(+KINK_DELTA):
            hi = refine_oracle(oenv, cp, ap, graphs[g], alpha=algo.alpha, max_iter=1)["action"]
        with shifted_relu_derivative(-KINK_DELTA):
            lo = refine_oracle(oenv, cp, ap, graphs[g], alpha=algo.alpha, max_iter=1)["action"]
        slack = 3.0 * ((hi - o1["action"]).abs() + (lo - o1["action"]).abs())
        assert float((err - slack).max()) <= 1e-4, (g, float(err.max()))
        n_kink += 1
    assert n_kink <= max(1, G // 3)


@pytest.mark.parametrize("env_id,N,G,area,n_obs,seed", CASES)
@pytest.mark.parametrize("pretrained", [True, False])
def test_full_loop_matches_float32_oracle(env_id, N, G, area, n_obs, seed, pretrained, gemm_path):
    G = 2 * G
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, seed + 10, pretrained)
    graph = _graph(env, agent, goal, pobs)
    a, v, it = _refine(algo, graph)
    packed = pobs.packed.cpu().numpy()
    o32 = _oracle_setup(env_id, N, area, n_obs, algo, agent, goal, packed, torch.float32)
    o64 = None
    n_close = n_multi = 0
    for g in range(G):
        o = refine_oracle(*o32[:3], o32[3][g], alpha=algo.alpha)
        n_dev = int(it[g]) & 0x3FFFFFFF
        assert (int(it[g]) >> 30 & 1) == (n_dev == 30 and float(v[g]) > 0)
        n_multi += n_dev > 1
        if n_dev == o["iters"]:
            np.testing.assert_allclose(a[g].numpy(), o["action"].double().numpy(), atol=2e-3, rtol=0, err_msg=f"graph {g}")
            if o["values"][-1] == o["values"][-1]:
                assert abs(float(v[g]) - o["values"][-1]) <= 2e-3 + 1e-2 * abs(o["values"][-1])
            continue
        # a different iteration count is excused only where float64 itself is within MARGIN of the decision
        if o64 is None:
            o64 = _oracle_setup(env_id, N, area, n_obs, algo, agent, goal, packed, torch.float64)
        r = refine_oracle(*o64[:3], o64[3][g], alpha=algo.alpha)
        k = min(n_dev, o["iters"]) - 1
        close = (k < len(r["values"]) and abs(r["values"][k]) < MARGIN) or bool((r["sel_term"].abs() < MARGIN).any())
        assert close, (g, n_dev, o["iters"], r["values"])
        n_close += 1
    assert n_close <= max(1, G // 4), f"{n_close} of {G} graphs decided within {MARGIN} of 0"


def _engine(env, algo, E, T, agent0, goal, pobs):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    eng = RolloutEngine(env, E, T=T, policy="actor_refine")
    eng.set_params(algo.actor_params)
    eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
    eng.set_initial(torch.from_numpy(agent0).cuda(), torch.from_numpy(goal).cuda(), pobs)
    return eng


@pytest.mark.parametrize("env_id,N,area,n_obs,seed", [("DoubleIntegrator", 6, 1.5, 2, 4), ("SingleIntegrator", 6, 1.5, 2, 8)])
def test_refined_rollout_matches_oracle_refinement(env_id, N, area, n_obs, seed, gemm_path):
    """Every step of a refined rollout against the oracle refining from the same state: the oracle's refined action
    and env.step from the rollout's state x_t must give the rollout's x_{t+1}.  (The closed loops themselves separate
    after the first step whose iteration count is decided by a value within rounding of 0 -- measured: 3e-3 after 5
    steps, 0.15 after 7 -- so the comparison is per step.)  Steps agree within 2e-4; at least a third of them must,
    some with more than one iteration.  A step may miss only where the device and the oracle took different iteration
    counts (counted; a minority) or where both stopped at the 30-iteration cap (at most a third): thirty gradient steps
    through ReLU kinks carry the rounding path of the oracle's float32 (measured: 3.2e-3 and 0.15 in x_{t+1}, the same
    on both GEMM paths to 1.4e-6), so there the recorded action must have lowered the loop value, by the oracle's
    evaluation.  Safe / finish / success rates of the
    rollout equal the oracle's masks evaluated on the same trajectory."""
    from oracle.algo import get_cbf, rates
    from refine_oracle import refine_value
    from gcbfplus_b200.trainer.utils import test_rates
    E, T = 2, 48
    env, algo, agent0, goal, pobs = _setup(env_id, N, E, area, n_obs, seed, True, vel_scale=0.0)
    eng = _engine(env, algo, E, T, agent0, goal, pobs)
    eng.run()
    torch.cuda.synchronize()
    st = eng.refine_stats()
    assert st["graph_steps"] == E * T and st["iters_max"] >= 1
    r, _, _ = test_rates(env, eng.result())
    states = eng.agent.cpu().numpy()
    actions = eng.actions.cpu().numpy()
    iters = eng.chains[0].refine_iters.cpu().numpy() & 0x3FFFFFFF
    packed = pobs.packed.cpu().numpy()
    oenv, cp, ap, _ = _oracle_setup(env_id, N, area, n_obs, algo, agent0, goal, packed, torch.float32)
    n_flip = n_multi = n_capped = n_strict = n_strict_multi = 0
    for e in range(E):
        obs = oracle_obstacles(packed[e], torch.float32)
        gl = torch.from_numpy(goal[e])
        col, fin = [], []
        for t in range(T + 1):
            g = oenv.get_graph(torch.from_numpy(states[t, e]), gl, obs)
            col.append(oenv.collision_mask(g))
            fin.append(oenv.finish_mask(g))
            if t == T:
                break
            o = refine_oracle(oenv, cp, ap, oenv.sparsify(g), alpha=algo.alpha)
            nxt, _, _ = oenv.step(g, o["action"])
            n_multi += int(iters[t, e]) > 1
            err = float(np.abs(nxt.agent.numpy() - states[t + 1, e]).max())
            if err <= 2e-4:
                n_strict += 1
                n_strict_multi += int(iters[t, e]) > 1
                continue
            if o["iters"] == int(iters[t, e]) == 30:
                # 30 steps through ReLU kinks: the capped iterate carries its rounding path (measured up to 0.15 in
                # x_{t+1}, identical on both GEMM paths), so it is held to what the loop promises: the recorded action
                # has a lower loop value than the loop's starting action, by the oracle's own evaluation
                gs = oenv.sparsify(g)
                h = get_cbf(cp, gs).squeeze(-1)
                with torch.no_grad():
                    v_dev = float(refine_value(oenv, cp, gs, h, torch.from_numpy(actions[t, e]), algo.alpha))
                assert v_dev < o["values"][0], (e, t, err, v_dev, o["values"][0], o["values"][-1])
                n_capped += 1
                continue
            assert o["iters"] != int(iters[t, e]), (e, t, err, o["iters"], int(iters[t, e]))
            n_flip += 1
        np.testing.assert_allclose(np.asarray(r[e], np.float64),
                                   rates(torch.stack(col).numpy(), torch.stack(fin).numpy()), atol=1e-6, rtol=0)
    assert n_multi > 0, "no step needed more than one refinement iteration: the test would not exercise the loop"
    assert n_flip <= E * T // 8, f"{n_flip} of {E * T} steps decided differently"
    # a third of the steps at least is compared at the strict tolerance, multi-iteration refinements among them;
    # steps that stopped at the cap on both sides are at most another third
    assert n_strict >= E * T // 3 and n_strict_multi > 0, (n_strict, n_strict_multi, n_capped, n_flip)
    assert n_capped <= E * T // 3, (n_strict, n_strict_multi, n_capped, n_flip)


def test_determinism(gemm_path):
    env_id, N, G, area, n_obs, seed = "DoubleIntegrator", 32, 6, 1.6, 6, 2
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, seed, True)
    graph = _graph(env, agent, goal, pobs)
    first = [x.clone() for x in algo.online_policy_refinement(graph, return_info=True)]
    second = algo.online_policy_refinement(graph, return_info=True)
    torch.cuda.synchronize()
    for x, y in zip(first, second):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    E, T = 3, 16
    a0, g0, _ = random_scene(env_id, N, E, 2.0, n_obs, seed=5)
    pobs2 = product_obstacles(env_id, random_scene(env_id, N, E, 2.0, n_obs, seed=5)[2])
    runs = []
    for _ in range(2):
        eng = _engine(env, algo, E, T, a0, g0, pobs2)
        eng.run()
        torch.cuda.synchronize()
        runs.append((eng.agent.clone(), eng.actions.clone(), eng.chains[0].refine_iters.clone()))
    for x, y in zip(*runs):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_refinement_follows_parameter_writes(gemm_path):
    """The optimizer and polyak kernels write parameters through raw pointers (torch sees no change).  Refinement
    after such a write must use the new CBF everywhere: bit-identical to a fresh object holding the new parameters.
    The rollout engine copies the CBF: it keeps the old one until set_cbf_params is called again."""
    from gcbfplus_b200 import _lib
    env_id, N, G, area, n_obs = "DoubleIntegrator", 12, 3, 1.2, 6
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, 9, True)
    other = product_algo(env, None, seed=5)
    graph = _graph(env, agent, goal, pobs)

    def refine(a):
        out = [x.clone() for x in a.online_policy_refinement(graph, return_info=True)]
        torch.cuda.synchronize()
        return out

    def same(x, y):
        return all(torch.equal(p.view(torch.int32), q.view(torch.int32)) for p, q in zip(x, y))

    def write_cbf():     # cbf <- (cbf + other's cbf) / 2 through the polyak kernel
        v = algo.cbf_params.flat._version
        _lib.check(env.lib.gcbf_polyak(_lib.ptr(algo.cbf_params.flat), _lib.ptr(other.cbf_params.flat),
                                       algo.cbf_params.count, 0.5, env._stream()), "gcbf_polyak")
        assert algo.cbf_params.flat._version == v

    E, T = 2, 8
    eng = _engine(env, algo, E, T, agent[:E], goal[:E], product_obstacles(env_id, random_scene(env_id, N, E, area,
                                                                                                  n_obs, 9)[2]))

    def roll():
        eng.run()
        torch.cuda.synchronize()
        return [eng.agent.clone(), eng.actions.clone(), eng.chains[0].refine_iters.clone()]

    before, roll0 = refine(algo), roll()
    write_cbf()
    after = refine(algo)
    fresh = product_algo(env, None, seed=7)
    fresh.cbf_params.flat.copy_(algo.cbf_params.flat)
    fresh.actor_net_params.flat.copy_(algo.actor_net_params.flat)
    assert same(after, refine(fresh))
    assert not same(after, before)
    assert same(roll(), roll0)                      # the engine's copy is unchanged by the write
    eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
    roll1 = roll()                                  # same captured graph, new CBF copy and planes
    assert not same(roll1, roll0)
    eng2 = _engine(env, fresh, E, T, agent[:E], goal[:E], product_obstacles(env_id, random_scene(env_id, N, E, area,
                                                                                                   n_obs, 9)[2]))
    eng2.run()
    torch.cuda.synchronize()
    assert same(roll1, [eng2.agent, eng2.actions, eng2.chains[0].refine_iters])


def test_nan_u_ref_stops_after_one_iteration(gemm_path):
    env_id, N, G, area, n_obs = "DoubleIntegrator", 8, 2, 1.2, 2
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, 7, True)
    goal[0, 3] = agent[0, 3]
    agent[0, 3, 2:] = 0.0
    goal[0, 3, 2:] = 0.0
    graph = _graph(env, agent, goal, pobs)
    a, v, it = _refine(algo, graph)
    assert int(it[0]) == 1 and np.isnan(float(v[0])), (int(it[0]), float(v[0]))
    assert (it[1:] & 0x3FFFFFFF).ge(1).all()
    oenv, cp, ap, graphs = _oracle_setup(env_id, N, area, n_obs, algo, agent, goal, pobs.packed.cpu().numpy(),
                                         torch.float32)
    o = refine_oracle(oenv, cp, ap, graphs[0], alpha=algo.alpha)
    assert o["iters"] == 1 and np.isnan(o["values"][0])
    assert torch.isnan(a[0, 3]).all()


def test_safe_batch_keeps_u_ref_and_takes_one_step(gemm_path):
    """Sparse scenes: every graph's value is 0 at the first iteration.  Agents with v_ref = 0 keep u_ref exactly, each
    graph takes its one mandatory step, and max_iter = 30 gives the same bits as max_iter = 1."""
    from gcbfplus_b200.algo.train import batch_u_ref
    env_id, N, G, area, n_obs = "DoubleIntegrator", 4, 4, 8.0, 0
    env, algo, agent, goal, pobs = _setup(env_id, N, G, area, n_obs, 11, True, vel_scale=0.0)
    graph = _graph(env, agent, goal, None)
    a30, v30, it30 = algo.online_policy_refinement(graph, return_info=True)
    a1, v1, it1 = algo.online_policy_refinement(graph, max_iter=1, return_info=True)
    ur = batch_u_ref(algo, {"agent": graph.agent, "goal": graph.goal})
    torch.cuda.synchronize()
    assert bool((v30 == 0).all()) and bool((it30 == 1).all()), (v30, it30)
    assert torch.equal(a30, a1) and torch.equal(v30, v1) and torch.equal(it30, it1)
    oenv, cp, ap, graphs = _oracle_setup(env_id, N, area, n_obs, algo, agent, goal, np.zeros((G, 0, 16), np.float32),
                                         torch.float64)
    for g in range(G):
        keep = ~refine_oracle(oenv, cp, ap, graphs[g], alpha=algo.alpha, max_iter=1)["sel"].numpy()
        assert keep.any()
        assert torch.equal(a30[g][torch.from_numpy(keep).cuda()], ur[g][torch.from_numpy(keep).cuda()])


def test_multi_layer_networks_are_rejected():
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env_id, N, G = "DoubleIntegrator", 4, 2
    env = product_env(env_id, N, 2.0, 0)
    deep = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, gnn_layers=2, seed=1)
    shallow = product_algo(env, env_id)
    agent, goal, _ = random_scene(env_id, N, G, 2.0, 0, seed=1)
    graph = _graph(env, agent, goal, None)
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        deep.online_policy_refinement(graph)
    with pytest.raises(NotImplementedError, match="actor has 2"):
        shallow.online_policy_refinement(graph, params=deep.actor_params)
    eng = RolloutEngine(env, G, T=4, policy="actor_refine")
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        eng.set_cbf_params(deep.cbf_params)
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        eng.set_params(deep.actor_params)
    with pytest.raises(ValueError, match="persistent"):
        RolloutEngine(env, G, T=4, policy="actor_refine", persistent=True)


def test_test_py_online_refine_end_to_end(tmp_path, capsys):
    """A run saved from the pretrained DoubleIntegrator npz, evaluated by test.py --path --online-refine."""
    import yaml
    env_id, N = "DoubleIntegrator", 6
    env = product_env(env_id, N, 1.5, 2)
    algo = product_algo(env, env_id)
    algo.save(str(tmp_path / "models"), 0)
    cfg = argparse.Namespace(env=env_id, num_agents=N, algo="gcbf+", buffer_size=algo.buffer_size, **algo.config)
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_refine_gpu", os.path.join(ROOT, "test.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    from train import build_parser
    args = build_parser(cli.FLAGS).parse_args(["--path", str(tmp_path), "--area-size", "1.5", "--obs", "2",
                                               "--epi", "3", "--max-step", "24", "--online-refine", "--no-video"])
    cli.test(args)
    out = capsys.readouterr().out
    assert "refinement iterations: median" in out and "of 72 graph-steps" in out
    assert "safe_rate" in out
    for bad in (["--env", env_id, "--u-ref"], ["--env", env_id, "--algo", "dec_share_cbf"]):
        with pytest.raises(SystemExit):
            cli.test(build_parser(cli.FLAGS).parse_args(bad + ["--area-size", "1.5", "--online-refine"]))
