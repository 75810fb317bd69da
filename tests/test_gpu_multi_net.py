"""GPU: several actor networks in one persistent rollout launch (gcbf_rollout_persistent_multi, RolloutEngine with
n_nets > 1).  Every network's environments must get the bits a solo persistent rollout of that network gives them:
states, LiDAR hits, actions, rewards, costs and per-step edge counts, whatever the network table's layout.  Where the
persistent kernel does not apply, the engine runs one solo engine per network; test.py --all-steps / --paths print, for
every network, the summary a solo test.py run prints."""
import argparse
import importlib.util
import os
import sys

import pytest
import torch

from helpers import ROOT, product_algo, product_env

pytestmark = pytest.mark.gpu

KEYS = ("agent", "hits", "actions", "rewards", "costs")
SCENES = {"SingleIntegrator": (8, 4.0, 0), "DoubleIntegrator": (16, 3.0, 6), "DubinsCar": (8, 2.5, 4)}


def _nets(env, env_id):
    """K = 3: two xavier networks with different seeds and the pretrained fixture."""
    return [product_algo(env, None, seed=s).actor_params for s in (1, 2)] + [product_algo(env, env_id).actor_params]


def _same(a, b):
    return torch.equal(a, b) or bool(((a == b) | (torch.isnan(a.float()) & torch.isnan(b.float()))).all())


def _record(eng, idx, k):
    """Network k's environments of a (batched or solo) engine's record, and its per-step edge counts / overflow."""
    out = {key: getattr(eng, key)[:, idx].clone() for key in KEYS}
    out["counters"] = eng.net_counters(k)[:, :2].clone()
    return out


def _solo(env, nets, k, idx, g0, T, n_obs, persistent=True):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    eng = RolloutEngine(env, len(idx), T=T, n_obs=n_obs, persistent=persistent)
    eng.set_params(nets[k])
    ix = torch.tensor(idx, device="cuda")
    eng.set_initial(g0.agent[ix], g0.goal[ix], g0.obstacle.select(idx) if n_obs > 0 else None)
    eng.run()
    torch.cuda.synchronize()
    return _record(eng, slice(None), 0)


def _compare_with_solo(env, eng, nets, g0, T, n_obs, persistent=True):
    for k, idx in enumerate(eng.net_envs):
        got, want = _record(eng, idx, k), _solo(env, nets, k, idx, g0, T, n_obs, persistent)
        for key in want:
            assert _same(got[key], want[key]), (k, key, float((got[key].float() - want[key].float()).abs().max()))


@pytest.mark.parametrize("layout", ["block", "interleaved"])
@pytest.mark.parametrize("env_id", list(SCENES))
def test_batched_launch_is_bit_identical_to_solo_launches(env_id, layout):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    N, area, n_obs = SCENES[env_id]
    E, T = 6, 32
    env = product_env(env_id, N, area, n_obs)
    g0 = env.reset(31, n_envs=E)        # a different initial state in every environment
    nets = _nets(env, env_id)
    table = None if layout == "block" else [g % 3 for g in range(E)]
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, persistent=True, n_nets=3, net_of_env=table)
    assert eng.persistent
    assert eng.net_envs == ([[0, 1], [2, 3], [4, 5]] if table is None else [[0, 3], [1, 4], [2, 5]])
    eng.set_params(nets)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    eng.run()                          # replay of the captured launch
    torch.cuda.synchronize()
    assert eng.launches_per_run == 1
    _compare_with_solo(env, eng, nets, g0, T, n_obs)
    # the networks really differ: the same initial state under two networks gives two trajectories
    a = eng.net_result(0).actions
    b = eng.net_result(1).actions
    assert not torch.equal(a, b)


def test_one_network_equals_the_single_network_entry_point():
    """K = 1: gcbf_rollout_persistent_multi with an all-zero table gives gcbf_rollout_persistent's bits."""
    import ctypes as C
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env_id = "DoubleIntegrator"
    N, area, n_obs = SCENES[env_id]
    E, T = 4, 32
    env = product_env(env_id, N, area, n_obs)
    g0 = env.reset(5, n_envs=E)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, persistent=True, use_cuda_graph=False)
    eng.set_params(product_algo(env, env_id).actor_params)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    want = {key: getattr(eng, key).clone() for key in KEYS}
    want["counters"] = eng.counters.clone()
    for key in KEYS:
        t = getattr(eng, key)
        (t[1:] if key == "agent" else t).fill_(float("nan"))
    counters = torch.zeros(T + 1, 1, 4, dtype=torch.int32, device="cuda")
    table = torch.zeros(E, dtype=torch.int32, device="cuda")
    rc = env.lib.gcbf_rollout_persistent_multi(
        C.byref(eng._pdesc), T, 1, eng.params_buf.data_ptr(), eng.infer_blob.data_ptr(), table.data_ptr(),
        eng.goal.data_ptr(), eng.obstacles.data_ptr(), env.ray_table.data_ptr(), eng.agent.data_ptr(),
        eng.hits.data_ptr(), eng.actions.data_ptr(), eng.rewards.data_ptr(), eng.costs.data_ptr(), counters.data_ptr(),
        eng._pws.data_ptr(), eng._pws.numel(), None, torch.cuda.current_stream().cuda_stream)
    _lib.check(rc, "gcbf_rollout_persistent_multi")
    torch.cuda.synchronize()
    for key in KEYS:
        assert _same(getattr(eng, key), want[key]), key
    assert torch.equal(counters[:, 0], want["counters"])


def test_more_clusters_than_resident_runs_in_rounds_with_the_same_bits():
    """A batched launch whose clusters are not all co-resident (gcbf_rollout_persistent_supported = 1, and too many
    CTAs for pair mode): the clusters beyond the resident ones run in later rounds and still give the solo bits."""
    import ctypes as C
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env_id = "DoubleIntegrator"
    N, area, n_obs, T = 8, 4.0, 8, 16
    env = product_env(env_id, N, area, n_obs)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per = sms // 3 + 1                 # 3 networks x per environments x 2 CTAs > 2 x the SM count
    E = 3 * per
    g0 = env.reset(7, n_envs=E)
    nets = _nets(env, env_id)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, n_nets=3)
    assert env.lib.gcbf_rollout_persistent_supported(C.byref(eng._pdesc)) == 1
    assert eng.persistent              # several networks take the persistent kernel at level 1 by default
    eng.set_params(nets)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    assert eng.launches_per_run == 1
    _compare_with_solo(env, eng, nets, g0, T, n_obs)


@pytest.mark.parametrize("case", ["LinearDrone", "two_layers"])
def test_fallback_runs_one_solo_engine_per_network(case):
    from gcbfplus_b200.algo.params import NetParams
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    if case == "LinearDrone":
        env_id, N, area, n_obs = "LinearDrone", 8, 1.2, 3
        env = product_env(env_id, N, area, n_obs)
        nets = [product_algo(env, None, seed=3).actor_params, product_algo(env, env_id).actor_params]
    else:
        env_id, (N, area, n_obs) = "DoubleIntegrator", SCENES["DoubleIntegrator"]
        env = product_env(env_id, N, area, n_obs)
        nets = [NetParams(env.edge_dim, env.action_dim, "actor", n_layers=2).init_xavier(s) for s in (4, 5)]
    E, T = 4, 24
    g0 = env.reset(13, n_envs=E)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, n_nets=2)
    eng.set_params(nets)
    assert not eng.persistent
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    _compare_with_solo(env, eng, nets, g0, T, n_obs, persistent=None)
    assert torch.equal(eng.counters[:, 0], eng._net_counters[:, :, 0].sum(dim=1))


# ------------------------------------------------------------------ test.py --all-steps / --paths
def _cli():
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_sweep_gpu", os.path.join(ROOT, "test.py"))
    cli = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(cli)
    return cli


def _save_run(run, env, env_id, algos_by_step):
    import yaml
    os.makedirs(run, exist_ok=True)
    for step, algo in algos_by_step.items():
        algo.save(os.path.join(run, "models"), step)
    algo = next(iter(algos_by_step.values()))
    cfg = argparse.Namespace(env=env_id, num_agents=env.num_agents, algo="gcbf+", buffer_size=algo.buffer_size,
                             **algo.config)
    with open(os.path.join(run, "config.yaml"), "w") as f:
        yaml.dump(cfg, f)


def _summary(out, prefix=""):
    return [l[len(prefix):] for l in out.splitlines() if l.startswith(prefix + "reward:")]


def test_test_py_all_steps_and_paths_match_solo_runs(tmp_path, capsys):
    env_id, N = "DoubleIntegrator", 8
    env = product_env(env_id, N, 2.0, 2)
    run_a, run_b = str(tmp_path / "run_a"), str(tmp_path / "run_b")
    _save_run(run_a, env, env_id, {0: product_algo(env, None, seed=1), 10: product_algo(env, None, seed=2),
                                   20: product_algo(env, None, seed=3)})
    _save_run(run_b, env, env_id, {7: product_algo(env, env_id)})
    cli = _cli()
    base = ["--area-size", "2.0", "--obs", "2", "--epi", "4", "--max-step", "32", "--no-video"]
    parse = cli.build_test_parser().parse_args

    def solo(run, step):
        cli.test(parse(["--path", run, "--step", str(step)] + base))
        lines = _summary(capsys.readouterr().out)
        assert len(lines) == 1
        return lines[0]

    cli.test(parse(["--path", run_a, "--all-steps", "--log"] + base))
    out = capsys.readouterr().out
    for step in (0, 10, 20):
        got = _summary(out, f"run={run_a} step={step} ")
        assert got == [solo(run_a, step)], step
    assert "best: run=" in out
    with open(os.path.join(run_a, "test_sweep.csv")) as f:
        rows = f.read().splitlines()
    assert [r.split(",")[0] for r in rows] == ["0", "10", "20"]
    assert not os.path.exists(os.path.join(run_a, "test_log.csv"))

    cli.test(parse(["--paths", run_a, run_b] + base))
    out = capsys.readouterr().out
    assert _summary(out, f"run={run_a} step=20 ") == [solo(run_a, 20)]
    assert _summary(out, f"run={run_b} step=7 ") == [solo(run_b, 7)]
    with capsys.disabled():
        print("\ntest.py --paths RUN_A RUN_B:")
        for line in out.splitlines():
            if line.startswith(("run=", "best:")):
                print("  " + line)
