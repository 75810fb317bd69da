"""GPU: observation and actuation noise of the rollout (csrc/noise.cu, RolloutEngine(perturbation=...)) against the
NumPy replica (tests/noise_oracle.py) and the oracle's closed loop, the sigma = 0 limits of every policy, one perturbed
step of every policy against that policy's own entry point, the invariances of the draws, and test.py's noise flags."""
import argparse
import ctypes as C
import importlib.util
import os
import sys

import numpy as np
import pytest
import torch

import noise_oracle as no
from helpers import ROOT, oracle_env, oracle_obstacles, oracle_params, product_algo, product_env

pytestmark = pytest.mark.gpu

REC = ("agent", "hits", "actions", "rewards", "costs")


def _ulps(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    ia = a.astype(np.float32).view(np.int32).astype(np.int64)
    ib = b.astype(np.float32).view(np.int32).astype(np.int64)
    ia = np.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = np.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return np.abs(ia - ib)


def test_normal_draws_match_replica():
    """10^6 draws of gcbf_normal_draws against the replica's fp32 z: equal, except where libm and CUDA's fp64 log / cos
    / sin round differently, by at most 1 fp32 ulp (the count is reported)."""
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(17)
    n = 250_000
    counters = np.zeros((n, 4), dtype=np.uint64)
    counters[:, 0] = rng.integers(0, 1024, n)
    counters[:, 1] = rng.integers(0, 2 ** 20, n)
    counters[:, 2] = rng.integers(0, 4096, n)
    counters[:, 3] = rng.integers(0, 2 ** 63, n, dtype=np.uint64) * np.uint64(2) + np.uint64(1)
    dev_c = torch.from_numpy(counters.view(np.int64)).cuda()
    total_diff = 0
    for seed, kind in ((1234, 0), (2 ** 64 - 5, 1), (7, 2)):
        out = torch.empty(n, 4, dtype=torch.float32, device="cuda")
        _lib.check(lib.gcbf_normal_draws(seed, kind, dev_c.data_ptr(), n, out.data_ptr(), None), "gcbf_normal_draws")
        torch.cuda.synchronize()
        got, want = out.cpu().numpy(), no.normals(seed, kind, counters)
        u = _ulps(got, want)
        assert u.max() <= 1, u.max()
        total_diff += int((u > 0).sum())
    print(f"\ngcbf_normal_draws: {total_diff} of {3 * 4 * n} draws differ from the replica by 1 fp32 ulp")
    assert total_diff <= 3 * 4 * n * 1e-4
    assert lib.gcbf_normal_draws(0, 3, dev_c.data_ptr(), 1, out.data_ptr(), None) < 0
    assert lib.gcbf_normal_draws(0, 0, None, 0, None, None) == 0


def _scene(env_id, N, E, area, n_obs, seed=11):
    env = product_env(env_id, N, area, n_obs)
    return env, env.reset(seed, n_envs=E)


@pytest.mark.parametrize("env_id,N,E,area,n_obs", [("DoubleIntegrator", 8, 3, 2.0, 4), ("LinearDrone", 8, 2, 1.2, 3)])
def test_perturb_kernels_match_replica(env_id, N, E, area, n_obs):
    """x + sigma z and h + sigma z bit for bit wherever the replica's z equals the device's; no-hit sentinels and
    components with sigma 0 are copied; the action noise in place."""
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.trainer.rollout import Perturbation
    env, g = _scene(env_id, N, E, area, n_obs)
    lib, d = env.lib, env.desc(E, n_obs)
    sd, nu = env.state_dim, env.action_dim
    sx = [0.05 * (k + 1) for k in range(sd)]
    sx[1] = 0.0
    su = [0.3] * nu
    p = Perturbation(sx, 0.07, su, seed=99, env_offset=4)
    buf = p.pack(env).cuda()
    obs_a, obs_h = torch.empty_like(g.agent), torch.empty_like(g.hits)
    for t in (0, 13):
        _lib.check(lib.gcbf_perturb_observation(C.byref(d), buf.data_ptr(), t, 4, g.agent.data_ptr(), g.hits.data_ptr(),
                                                obs_a.data_ptr(), obs_h.data_ptr(), None), "gcbf_perturb_observation")
        act = torch.randn(E, env.num_agents, nu, device="cuda")
        act0 = act.clone()
        _lib.check(lib.gcbf_perturb_action(C.byref(d), buf.data_ptr(), t, 4, act.data_ptr(), None), "gcbf_perturb_action")
        torch.cuda.synchronize()
        x, h = g.agent.cpu().numpy(), g.hits.cpu().numpy()
        env_ids = [4 + e for e in range(E)]
        want_x, want_h = no.observe(99, t, env_ids, x, h, sx, 0.07, env.params["comm_radius"])
        want_a = no.act_noise(99, t, env_ids, act0.cpu().numpy(), su)
        for got, want in ((obs_a, want_x), (obs_h, want_h), (act, want_a)):
            got = got.cpu().numpy()
            same = got.view(np.int32) == want.view(np.int32)
            # a 1-ulp z difference moves x + sigma z by at most sigma ulp(z) (+ the rounding of the sum)
            assert same.mean() > 0.999 and np.abs(got - want)[~same].max(initial=0) <= 1e-6, (same.mean(),)
        assert np.array_equal(obs_a.cpu().numpy()[..., 1].view(np.int32), x[..., 1].view(np.int32))   # sigma 0: copied
        miss = np.sqrt(((h - x[:, :, None, :h.shape[-1]]) ** 2).sum(-1)) > 1e3
        assert miss.any() and (~miss).any()
        assert np.array_equal(obs_h.cpu().numpy()[miss].view(np.int32), h[miss].view(np.int32))
        assert (obs_h.cpu().numpy()[~miss] != h[~miss]).mean() > 0.99
    # argument checks
    assert lib.gcbf_perturb_observation(C.byref(d), buf.data_ptr(), -1, 0, g.agent.data_ptr(), g.hits.data_ptr(),
                                        obs_a.data_ptr(), obs_h.data_ptr(), None) < 0
    assert lib.gcbf_perturb_observation(C.byref(d), buf.data_ptr(), 0, 0, g.agent.data_ptr(), g.hits.data_ptr(),
                                        g.agent.data_ptr(), obs_h.data_ptr(), None) < 0
    assert lib.gcbf_perturb_action(C.byref(d), buf.data_ptr() + 4, 0, 0, act.data_ptr(), None) < 0


def _oracle_noisy_rollout(oenv, ap, agent0, goal0, obstacles, T, seed, env_id, sx, sl, su, comm_radius):
    """The oracle's closed loop under the perturbation model: the true graph, add_edge_feats with the observed states
    (x_hat | goal | h_hat), act, + sigma_u z, env.step of the true state."""
    from oracle.nn import net_forward
    N, R, pd = oenv.num_agents, oenv.n_hits, oenv.pos_dim
    g = oenv.get_graph(agent0, goal0, obstacles)
    states, actions, rewards, collide, finish = [], [], [], [], []
    with torch.no_grad():
        for t in range(T):
            gs = oenv.sparsify(g)
            lid = g.states[2 * N:2 * N + N * R].clone()
            x_hat, h_hat = no.observe(seed, t, [env_id], g.agent.numpy()[None],
                                      lid[:, :pd].numpy().reshape(1, N, R, pd), sx, sl, comm_radius)
            lid[:, :pd] = torch.from_numpy(h_hat.reshape(N * R, pd))
            xh = torch.from_numpy(x_hat[0])
            go = oenv.add_edge_feats(gs, torch.cat([xh, g.goal, lid], dim=0))
            a = 2 * net_forward(ap, go, "actor") + oenv.u_ref(xh, g.goal)
            a = torch.from_numpy(no.act_noise(seed, t, [env_id], a.numpy()[None], su)[0])
            states.append(g.agent)
            collide.append(oenv.collision_mask(g))
            finish.append(oenv.finish_mask(g))
            g, r, _ = oenv.step(g, a)
            actions.append(a)
            rewards.append(r)
        states.append(g.agent)
        collide.append(oenv.collision_mask(g))
        finish.append(oenv.finish_mask(g))
    return {"states": torch.stack(states), "actions": torch.stack(actions), "rewards": torch.stack(rewards),
            "collision": torch.stack(collide), "finish": torch.stack(finish)}


def _as_rollout_result(res):
    from gcbfplus_b200.env.base import RolloutResult
    g = {"agent": res.agent.transpose(0, 1).contiguous(), "goal": res.goal, "hits": res.hits.transpose(0, 1).contiguous(),
         "obstacle": res.obstacle}
    return RolloutResult(g, res.actions.transpose(0, 1), res.rewards.transpose(0, 1), res.costs.transpose(0, 1),
                         res.dones.transpose(0, 1), {})


@pytest.mark.parametrize("env_id,N,E,area,n_obs", [("DoubleIntegrator", 8, 2, 2.0, 4), ("DubinsCar", 8, 2, 2.5, 4),
                                                    ("SingleIntegrator", 8, 2, 2.0, 0), ("LinearDrone", 8, 2, 1.2, 3)])
def test_noisy_rollout_matches_oracle(env_id, N, E, area, n_obs, gemm_path):
    """The perturbed actor rollout against the oracle's noisy closed loop over 24 steps: the tolerance of the noiseless
    rollout-versus-oracle test (test_gpu_rollout.py: first step, the first quarter, the whole window), identical safe /
    finish / success rates."""
    from gcbfplus_b200.trainer.rollout import Perturbation, RolloutEngine
    from oracle.algo import rates
    T, seed, off = 24, 31, 5
    env, g0 = _scene(env_id, N, E, area, n_obs)
    sx, sl, su = [0.02] * env.state_dim, 0.02, [0.1] * env.action_dim
    algo = product_algo(env, env_id)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, perturbation=Perturbation(sx, sl, su, seed, env_offset=off))
    assert not eng.persistent
    eng.set_params(algo.actor_params)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    res = eng.result()
    col, fin = env.rollout_masks(_as_rollout_result(res))
    oenv = oracle_env(env_id, N, area, n_obs)
    ap, _ = oracle_params(env_id)
    packed = g0.obstacle.packed.cpu().numpy() if n_obs > 0 else np.zeros((E, 0, 16), np.float32)
    for e in range(E):
        ref = _oracle_noisy_rollout(oenv, ap, g0.agent[e].cpu(), g0.goal[e].cpu(), oracle_obstacles(packed[e]), T, seed,
                                    off + e, sx, sl, su, env.params["comm_radius"])
        err = np.abs(res.agent[e].cpu().numpy() - ref["states"].numpy()).reshape(T + 1, -1).max(axis=1)
        assert err[1] <= (2e-6 if gemm_path == "simt" else 6e-6), err[:4]
        assert err[:T // 4].max() <= (1e-4 if gemm_path == "simt" else 3e-4), err[:T // 4].max()
        assert err.max() <= 5e-3, err.max()
        aerr = np.abs(res.actions[e].cpu().numpy() - ref["actions"].numpy()).reshape(T, -1).max(axis=1)
        assert aerr[0] <= 1e-4, aerr[:4]      # identical inputs at t = 0: the network's rounding only
        np.testing.assert_allclose(res.rewards[e].cpu().numpy(), ref["rewards"].numpy(), atol=5e-3)
        got = rates(col[:, e].cpu().numpy(), fin[:, e].cpu().numpy())
        want = rates(ref["collision"].numpy(), ref["finish"].numpy())
        assert got == want, (got, want)
    # the observation the engine recorded is x + sigma z of the true states (t = 0: identical inputs)
    x_hat, _ = no.observe(seed, 0, [off + e for e in range(E)], g0.agent.cpu().numpy(), g0.hits.cpu().numpy(), sx, sl,
                          env.params["comm_radius"])
    assert np.abs(eng.obs_agent[0].cpu().numpy() - x_hat).max() <= 1e-6


def _engine(env, g0, E, T, n_obs, policy, algo, perturbation=None, **kw):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, policy=policy, perturbation=perturbation, **kw)
    if policy in ("actor", "actor_refine", "actor_qp", "u_ref_qp"):
        eng.set_params(algo.actor_params)
    if policy in ("actor_refine", "actor_qp", "u_ref_qp"):
        eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    return eng


POLICIES = ("actor", "u_ref", "actor_refine", "actor_qp", "u_ref_qp", "dec_share_cbf", "centralized_cbf")


@pytest.mark.parametrize("policy", POLICIES)
def test_zero_sigma_equals_noiseless_rollout(policy):
    """sigma = 0: the refinement, both safety filters and both baselines give the noiseless rollout's bits.  The actor
    moves from the fused step to the modular sequence with every edge feature clipped, u_ref from env_step mode 2 to
    gcbf_act + mode 1: those agree to closed-loop rounding, with identical rates (the largest difference is reported)."""
    from gcbfplus_b200.trainer.rollout import Perturbation
    from oracle.algo import rates
    env_id, N, E, area, n_obs, T = "DoubleIntegrator", 8, 3, 2.0, 4, 24
    env, g0 = _scene(env_id, N, E, area, n_obs)
    algo = product_algo(env, env_id)
    outs = []
    for pert in (None, Perturbation(0.0, 0.0, 0.0, seed=5)):
        eng = _engine(env, g0, E, T, n_obs, policy, algo, pert, persistent=False)
        eng.run()
        torch.cuda.synchronize()
        outs.append((eng, {k: getattr(eng, k).clone() for k in REC}))
    (e0, a), (e1, b) = outs
    assert torch.equal(e1.obs_agent, e1.agent[:-1])
    if policy in ("actor", "u_ref"):
        diff = max(float((a[k] - b[k]).abs().nan_to_num().max()) for k in ("agent", "actions"))
        print(f"\n{policy}: sigma = 0 vs noiseless, largest state / action difference over {T} steps: {diff:.3g}")
        assert diff <= 3e-4
        ca, fa = env.rollout_masks(_as_rollout_result(e0.result()))
        cb, fb = env.rollout_masks(_as_rollout_result(e1.result()))
        for e in range(E):
            assert rates(ca[:, e].cpu().numpy(), fa[:, e].cpu().numpy()) == rates(cb[:, e].cpu().numpy(),
                                                                                 fb[:, e].cpu().numpy())
        return
    for k in REC:
        assert torch.equal(a[k], b[k]) or bool(((a[k] == b[k]) | (a[k].isnan() & b[k].isnan())).all()), k


@pytest.mark.parametrize("policy", POLICIES)
def test_one_perturbed_step_equals_policy_entry(policy):
    """sigma > 0, one step: the recorded observation is the replica's x_hat, and the recorded action is the policy's own
    entry point called on the observed graph (the step's true edges, x_hat and h_hat) plus the replica's action noise."""
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.trainer.rollout import Perturbation
    from gcbfplus_b200.utils.graph import SwarmGraph
    env_id, N, E, area, n_obs = "DoubleIntegrator", 8, 2, 2.0, 4
    env, g0 = _scene(env_id, N, E, area, n_obs, seed=3)
    algo = product_algo(env, env_id)
    sx, sl, su, seed, off = [0.03, 0.02, 0.05, 0.04], 0.03, [0.2, 0.1], 77, 2
    eng = _engine(env, g0, E, 1, n_obs, policy, algo, Perturbation(sx, sl, su, seed, env_offset=off))
    eng.run()
    torch.cuda.synchronize()
    ids = [off + e for e in range(E)]
    x_hat, h_hat = no.observe(seed, 0, ids, eng.agent[0].cpu().numpy(), eng.hits[0].cpu().numpy(), sx, sl,
                              env.params["comm_radius"])
    assert np.abs(eng.obs_agent[0].cpu().numpy() - x_hat).max() <= 1e-6
    assert np.abs(np.nan_to_num(eng._obs_hits.cpu().numpy() - h_hat)).max() <= 1e-6
    ch, lib, nu = eng.chains[0], env.lib, env.action_dim
    graph = SwarmGraph(env, torch.from_numpy(x_hat).cuda(), eng.goal, g0.obstacle, torch.from_numpy(h_hat).cuda(),
                       ch.row_start[0], ch.row_deg[0], ch.edge_recv[0], ch.edge_src[0], ch.counters[0])
    args = (graph.agent, graph.goal, graph.hits, graph.row_start, graph.row_deg, graph.edge_recv, graph.edge_src,
            graph.counters)
    d = ch.desc

    def pi(clip_all):     # the rollout's policy forward: folded weights (gcbf_gnn_infer)
        out = torch.empty(E, N, nu, device="cuda")
        _lib.check(lib.gcbf_gnn_infer(C.byref(d), _lib.NET_ACTOR, nu, eng.params_buf.data_ptr(),
                                      eng.infer_blob.data_ptr(), eng.use_tc, *[_lib.ptr(x) for x in args], clip_all,
                                      out.data_ptr(), ch.ws.data_ptr(), ch.ws.numel(), None), "gcbf_gnn_infer")
        return out

    def act(p):           # gcbf_act: 2 pi + u_ref(x_hat), or u_ref(x_hat)
        out = torch.empty(E, N, nu, device="cuda")
        _lib.check(lib.gcbf_act(C.byref(d), graph.agent.data_ptr(), graph.goal.data_ptr(), _lib.ptr(p), out.data_ptr(),
                                None), "gcbf_act")
        return out

    if policy == "actor":
        cmd = act(pi(1))
    elif policy == "u_ref":
        cmd = act(None)
    elif policy == "actor_refine":
        from gcbfplus_b200.algo.refine import launch_refine, refine_workspace
        cmd = torch.empty(E, N, nu, device="cuda")
        iters = torch.empty(E, dtype=torch.int32, device="cuda")
        launch_refine(env, d, eng.refine_alpha, eng.refine_lr, eng.refine_max_iter, eng.use_tc, eng.cbf_params,
                      eng._refine_planes, pi(0), *args, cmd, None, iters, refine_workspace(env, d), None)
    elif policy == "actor_qp":
        cmd = algo.safety_filter(graph, u_nom=act(pi(0)))
    elif policy == "u_ref_qp":
        cmd = algo.safety_filter(graph)
    else:
        cmd = eng.controller.act(graph)
    torch.cuda.synchronize()
    want = no.act_noise(seed, 0, ids, cmd.cpu().numpy(), su)
    got = eng.actions[0].cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(np.nan_to_num(got).view(np.int32), np.nan_to_num(want).view(np.int32)), \
        float(np.nanmax(np.abs(got - want)))


def test_draws_are_invariant_to_batch_offset_and_capture():
    """The same seed gives the same bits; episode 5 gets the same trajectory as environment 5 of 8 and as environment 2 of
    the batch of episodes 3..7 (env_offset 3), with and without a CUDA graph; set_perturbation changes the sigmas of a
    captured rollout without a new capture."""
    from gcbfplus_b200.trainer.rollout import Perturbation
    from gcbfplus_b200.utils import jrandom as jr
    env_id, N, area, n_obs, T = "DoubleIntegrator", 8, 4.0, 4, 32
    env = product_env(env_id, N, area, n_obs)
    algo = product_algo(env, env_id)
    keys = jr.split(jr.PRNGKey(1234), 1_000)[:8]
    runs = []
    for offset, graph_on in ((0, True), (0, True), (3, True), (3, False)):
        g0 = env.reset(jr.split(keys[offset:], 2)[:, 0])
        p = Perturbation(0.02, 0.02, 0.1, seed=1234, env_offset=offset)
        eng = _engine(env, g0, 8 - offset, T, n_obs, "actor", algo, p, use_cuda_graph=graph_on)
        eng.run()
        torch.cuda.synchronize()
        runs.append({k: getattr(eng, k).clone() for k in REC + ("obs_agent",)})
        if offset == 0 and graph_on and len(runs) == 1:
            captured = eng
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k
        assert torch.equal(runs[0][k][:, 5], runs[2][k][:, 2]), k
        assert torch.equal(runs[2][k], runs[3][k]), k
    graph = captured._graph
    p2 = Perturbation(0.05, 0.0, [0.2, 0.0], seed=9)
    captured.set_perturbation(p2)
    captured.run()
    assert captured._graph is graph
    g0 = env.reset(jr.split(keys, 2)[:, 0])
    fresh = _engine(env, g0, 8, T, n_obs, "actor", algo, p2)
    fresh.run()
    torch.cuda.synchronize()
    for k in REC:
        assert torch.equal(getattr(captured, k), getattr(fresh, k)), k
    assert not torch.equal(captured.actions, runs[0]["actions"])


def test_test_py_noise_end_to_end(tmp_path, capsys):
    """A run saved from the pretrained DoubleIntegrator npz, evaluated by test.py with and without noise on the same
    five episodes.  Both safe rates are reported; the noisy one is expected to be lower but is not asserted."""
    import yaml
    env_id, N = "DoubleIntegrator", 8
    env = product_env(env_id, N, 4.0, 8)
    algo = product_algo(env, env_id)
    algo.save(str(tmp_path / "models"), 0)
    cfg = argparse.Namespace(env=env_id, num_agents=N, algo="gcbf+", buffer_size=algo.buffer_size, **algo.config)
    with open(tmp_path / "config.yaml", "w") as f:
        yaml.dump(cfg, f)
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_noise_gpu", os.path.join(ROOT, "test.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    base = ["--path", str(tmp_path), "--area-size", "4", "--epi", "5", "--no-video", "--log"]
    noise = ["--state-noise", "0.02", "--lidar-noise", "0.02", "--action-noise", "0.1"]
    lines = {}
    for name, extra in (("noiseless", []), ("noisy", noise)):
        cli.test(cli.build_test_parser().parse_args(base + extra))
        out = capsys.readouterr().out
        lines[name] = [l for l in out.splitlines() if l.startswith(("reward:", "noise:"))]
        assert any("safe_rate" in l for l in lines[name])
    assert any(l.startswith("noise: state sigma [0.02, 0.02, 0.02, 0.02], LiDAR sigma 0.02, action sigma [0.1, 0.1]")
               for l in lines["noisy"])
    with capsys.disabled():
        for name, ls in lines.items():
            print(f"\ntest.py {name}:")
            for l in ls:
                print("  " + l)
    with open(tmp_path / "test_log.csv") as f:
        assert len(f.read().splitlines()) == 1
    with open(tmp_path / "test_log_noise.csv") as f:
        rows = f.read().splitlines()
    assert len(rows) == 1 and rows[0].startswith("0.02 0.02 0.02 0.02,0.02,0.1 0.1,1234,8,5,")
