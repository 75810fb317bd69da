"""GPU parity: closed-loop rollout (CUDA-graph engine) vs the oracle's rollout from identical
initial conditions with the reference's pretrained weights.  Bar (SURVEY 8c): trajectories
within a tolerance that grows with t (chaotic closed loop, fp32 summation order), safe / finish /
success rates (test.py:184-198) identical."""
import numpy as np
import pytest
import torch

from helpers import (oracle_env, oracle_obstacles, oracle_params, product_algo, product_env, random_scene)

pytestmark = pytest.mark.gpu


def _reset_scene(env_id, N, E, area, n_obs, seed):
    env = product_env(env_id, N, area, n_obs)
    graph = env.reset(seed, n_envs=E)
    return env, graph


@pytest.mark.parametrize("env_id,N,E,area,n_obs,T", [("DoubleIntegrator", 8, 3, 2.0, 4, 96),
                                                      # BASELINE.json configs[0] literally: SingleIntegrator n=8, area-size 4,
                                                      # 16 envs, obs 0, full 256-step episode
                                                      ("SingleIntegrator", 8, 16, 4.0, 0, 256),
                                                      # configs[1] literally: DoubleIntegrator n=8, 16 envs (PARAMS default 8 obstacles)
                                                      ("DoubleIntegrator", 8, 16, 4.0, 8, 256),
                                                      ("SingleIntegrator", 8, 2, 2.0, 4, 64),
                                                      ("DubinsCar", 8, 2, 2.5, 4, 64),
                                                      ("LinearDrone", 8, 2, 1.2, 3, 48)])
def test_rollout_matches_oracle(env_id, N, E, area, n_obs, T, gemm_path):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    from oracle.algo import rates, rollout
    env, g0 = _reset_scene(env_id, N, E, area, n_obs, seed=11)
    algo = product_algo(env, env_id)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs)
    eng.set_params(algo.actor_params)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    first = {k: getattr(eng, k).clone() for k in ("agent", "hits", "actions", "rewards", "costs")}
    eng.run()                                   # CUDA-graph replay must be bit-reproducible
    torch.cuda.synchronize()
    for k, v in first.items():
        assert torch.equal(v, getattr(eng, k)) or (torch.isnan(v) == torch.isnan(getattr(eng, k))).all(), k
    # eager (no graph) engine gives the same bits
    eng2 = RolloutEngine(env, E, T=T, n_obs=n_obs, use_cuda_graph=False)
    eng2.set_params(algo.actor_params)
    eng2.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng2.run()
    torch.cuda.synchronize()
    assert torch.equal(eng2.agent, eng.agent)
    res = eng.result()
    col, fin = env.rollout_masks(_as_rollout_result(res))
    oenv = oracle_env(env_id, N, area, n_obs)
    ap, _ = oracle_params(env_id)
    packed = g0.obstacle.packed.cpu().numpy()
    for e in range(E):
        ref = rollout(oenv, ap, g0.agent[e].cpu(), g0.goal[e].cpu(), oracle_obstacles(packed[e]), T=T)
        got = res.agent[e].cpu().numpy()
        want = ref["states"].numpy()
        err = np.abs(got - want).reshape(T + 1, -1).max(axis=1)
        assert err[1] <= (2e-6 if gemm_path == "simt" else 6e-6), err[:4]
        # closed-loop drift over the first steps (T/4, at most 24: the window the bound was calibrated on -- the loop is
        # chaotic, a 256-step episode measured 6.7e-4 at step 62): the per-step network tolerance (1e-5 SIMT / 3e-5
        # tensor core, test_gpu_gnn.py) amplified by the closed loop -- same 3x ratio between the two paths
        w = min(T // 4, 24)
        assert err[:w].max() <= (1e-4 if gemm_path == "simt" else 3e-4), err[:w].max()
        assert err.max() <= 5e-3, err.max()
        np.testing.assert_allclose(res.rewards[e].cpu().numpy(), ref["rewards"].numpy(), atol=5e-3)
        got_rates = rates(col[:, e].cpu().numpy(), fin[:, e].cpu().numpy())
        want_rates = rates(ref["collision"].numpy(), ref["finish"].numpy())
        assert got_rates == want_rates, (got_rates, want_rates)


def _as_rollout_result(res):
    from gcbfplus_b200.env.base import RolloutResult
    g = {"agent": res.agent.transpose(0, 1).contiguous(), "goal": res.goal, "hits": res.hits.transpose(0, 1).contiguous(),
         "obstacle": res.obstacle}
    return RolloutResult(g, res.actions.transpose(0, 1), res.rewards.transpose(0, 1), res.costs.transpose(0, 1),
                         res.dones.transpose(0, 1), {})


@pytest.mark.parametrize("env_id,N,E,area,n_obs,T", [("DoubleIntegrator", 48, 3, 3.0, 6, 12), ("SingleIntegrator", 8, 16, 4.0, 0, 40),
                                                      ("DubinsCar", 12, 2, 2.0, 4, 24), ("DoubleIntegrator", 200, 2, 6.0, 8, 8),
                                                      ("DoubleIntegrator", 130, 1, 4.0, 3, 6),
                                                      ("DoubleIntegrator", 512, 3, 16.0, 8, 5),
                                                      # BASELINE configs[2] shape: 16 environments x 8 CTAs (pair mode where
                                                      # fewer than 16 hardware clusters of 8 are resident)
                                                      ("DoubleIntegrator", 512, 16, 32.0, 8, 4)])
def test_persistent_rollout_is_bit_identical_to_5_launch_path(env_id, N, E, area, n_obs, T):
    """The single-launch persistent rollout (one thread-block cluster per environment, csrc/rollout_persist.cu) against
    the 5-launch env-step path: same operand splits, MMA order, epilogues and reduction orders -> the same bits for
    states, LiDAR hits, actions, rewards, costs and per-step edge counts (dense scenes: several edge tiles per CTA,
    ragged last tiles, N not a multiple of the cluster size)."""
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env, g0 = _reset_scene(env_id, N, E, area, n_obs, seed=21)
    algo = product_algo(env, env_id)
    outs = []
    for persistent in (True, False):
        eng = RolloutEngine(env, E, T=T, n_obs=n_obs, persistent=persistent)
        assert eng.persistent == persistent
        eng.set_params(algo.actor_params)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        eng.run()
        eng.run()                                   # replay of the captured launch
        torch.cuda.synchronize()
        outs.append({k: getattr(eng, k).clone() for k in ("agent", "hits", "actions", "rewards", "costs")})
        outs[-1]["n_edges"] = eng.counters[:, 0].clone()
        assert eng.launches_per_run == (1 if persistent else 1 + 5 * T)
    for k in outs[0]:
        a, b = outs[0][k], outs[1][k]
        if env_id == "DubinsCar" and k != "n_edges":
            # DubinsCar agrees to closed-loop rounding only: identical while all speeds are 0, then a few policy outputs
            # differ by 1-2 ulp per step (the heading's sin / cos enter
            # the edge features in two translation units) -> 1.6e-5 after 24 steps.  RolloutEngine therefore does not
            # pick the persistent kernel for DubinsCar by default
            if k != "hits":          # (missed rays sit 1e6 ranges away: their ulp is 0.03)
                assert float((a.float() - b.float()).abs().nan_to_num().max()) <= 2e-4, k
            continue
        same = torch.equal(a, b) or bool(((a == b) | (torch.isnan(a.float()) & torch.isnan(b.float()))).all())
        assert same, (k, float((a.float() - b.float()).abs().nan_to_num().max()))


def _persist_digest(n_agents=200, n_envs=2, T=8):
    """sha256 of a persistent-kernel rollout's record (this or a child process)."""
    import hashlib
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env, g0 = _reset_scene("DoubleIntegrator", n_agents, n_envs, 6.0, 8, seed=21)
    algo = product_algo(env, "DoubleIntegrator")
    eng = RolloutEngine(env, n_envs, T=T, n_obs=8, persistent=True)
    eng.set_params(algo.actor_params)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    eng.run()
    torch.cuda.synchronize()
    h = hashlib.sha256()
    for t in (eng.agent, eng.hits, eng.actions, eng.rewards, eng.costs, eng.counters[:, 0]):
        h.update(t.cpu().numpy().tobytes())
    return h.hexdigest()


def test_persistent_soft_groups_equal_hardware_clusters():
    """The persistent kernel's two synchronisation modes -- hardware thread-block clusters (barrier.cluster + DSMEM) and
    software groups of a cooperative launch (global arrival counters; what 16 environments x 8 CTAs need on a device
    where fewer than 16 such clusters are resident at once) -- must produce the same bits."""
    import os
    import subprocess
    import sys
    here = os.path.dirname(os.path.abspath(__file__))
    code = ("import sys; sys.path.insert(0, %r); sys.path.insert(0, %r); import test_gpu_rollout as t; "
            "print('DIGEST', t._persist_digest())" % (here, os.path.dirname(here)))
    out = subprocess.run([sys.executable, "-c", code], env=dict(os.environ, GCBF_PERSIST_SOFT="1"), capture_output=True,
                         text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-2000:]
    other = [l for l in out.stdout.splitlines() if l.startswith("DIGEST")][0].split()[1]
    assert other == _persist_digest()
