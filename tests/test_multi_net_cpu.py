"""CPU: the multi-network persistent rollout's C entry point and stride query (exported, argument checks without a
device), the engine's host validation of the network table and the networks, and test.py's --all-steps / --paths flag
handling."""
import argparse
import ctypes
import importlib.util
import os
import sys
import types

import pytest

from helpers import ROOT


def _desc(kind=1, G=4, N=8, R=32, O=0):
    from gcbfplus_b200 import _lib
    d = _lib.EnvDesc()
    d.env_kind, d.n_graphs, d.n_agents, d.n_rays, d.n_hits, d.n_obs = kind, G, N, R, R, O
    d.edge_cap, d.obs_per_graph = G * N * 48, 1
    return d


def test_multi_symbols_exported_and_bound():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    for n in ("gcbf_rollout_persistent_multi", "gcbf_rollout_persistent_multi_strides"):
        assert hasattr(lib, n), n
        assert n in _lib._SIGNATURES, n


def test_strides_are_the_counts_rounded_to_16_bytes():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    for ed, nu in ((2, 2), (4, 2), (6, 3)):
        ps, ist = ctypes.c_int64(), ctypes.c_int64()
        assert lib.gcbf_rollout_persistent_multi_strides(ed, nu, ctypes.byref(ps), ctypes.byref(ist)) == 0
        pc, ic = lib.gcbf_param_count_l(ed, nu, 1), lib.gcbf_infer_count(ed, nu)
        assert ps.value == (pc + 3) // 4 * 4 and ist.value == (ic + 3) // 4 * 4
    ps, ist = ctypes.c_int64(), ctypes.c_int64()
    assert lib.gcbf_rollout_persistent_multi_strides(9, 2, ctypes.byref(ps), ctypes.byref(ist)) < 0
    assert b"bad argument" in lib.gcbf_last_error_string()
    assert lib.gcbf_rollout_persistent_multi_strides(2, 2, None, None) < 0


def _call(lib, d, n_nets=2, params=None, blob=None, table=None, goal=None):
    p = ctypes.c_void_p(16)   # never dereferenced: every call below fails its argument checks first
    params = p if params is None else params
    blob = p if blob is None else blob
    table = p if table is None else table
    goal = p if goal is None else goal
    return lib.gcbf_rollout_persistent_multi(ctypes.byref(d), 4, n_nets, params, blob, table, goal, None, p, p, p, p,
                                             p, p, p, p, 1 << 30, None, None)


def test_multi_argument_errors_without_gpu():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    d = _desc()
    for n_nets in (0, -3):
        assert _call(lib, d, n_nets=n_nets) < 0
        assert b"n_nets must be >= 1" in lib.gcbf_last_error_string()
    assert _call(lib, d, table=ctypes.c_void_p(0)) < 0
    assert b"net_of_env is NULL" in lib.gcbf_last_error_string()
    for kw in ({"params": ctypes.c_void_p(20)}, {"blob": ctypes.c_void_p(24)}, {"table": ctypes.c_void_p(18)}):
        assert _call(lib, d, **kw) < 0
        assert b"16-byte aligned" in lib.gcbf_last_error_string(), kw
    # what gcbf_rollout_persistent rejects: NULL arrays, unsupported configurations
    assert _call(lib, d, goal=ctypes.c_void_p(0)) < 0
    assert b"gcbf_rollout_persistent_multi: NULL pointer argument" in lib.gcbf_last_error_string()
    for bad in (_desc(N=600), _desc(kind=3), _desc(O=40)):
        assert _call(lib, bad) < 0
        assert b"gcbf_rollout_persistent_multi: unsupported configuration" in lib.gcbf_last_error_string()


def test_engine_validates_the_network_table():
    from gcbfplus_b200.trainer.rollout import check_net_table
    assert check_net_table([0, 1, 2, 0, 1, 2], 3, 6) == [0, 1, 2, 0, 1, 2]
    for table, what in (([0, 1, 3, 0], "out of range"), ([0, -1, 1, 0], "out of range"), ([0, 1, 0], "3 entries"),
                        ([0, 0, 0, 0], "network 1 runs no environment")):
        with pytest.raises(ValueError, match=what):
            check_net_table(table, 2, 4)


def test_engine_refuses_uneven_blocks_and_other_policies_before_allocating():
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env = types.SimpleNamespace(max_episode_steps=8, params={"n_obs": 0}, enable_stop=True)
    with pytest.raises(ValueError, match="multiple of n_nets"):
        RolloutEngine(env, 10, n_nets=4)
    with pytest.raises(ValueError, match="n_nets must be >= 1"):
        RolloutEngine(env, 4, n_nets=0)
    for policy in ("u_ref", "actor_refine", "actor_qp"):
        with pytest.raises(ValueError, match="policy 'actor'"):
            RolloutEngine(env, 4, policy=policy, n_nets=2)
    with pytest.raises(ValueError, match="out of range"):
        RolloutEngine(env, 4, n_nets=2, net_of_env=[0, 1, 2, 0])


def test_engine_refuses_mixed_networks():
    from gcbfplus_b200.algo.params import NetParams
    from gcbfplus_b200.trainer.rollout import check_nets
    a = NetParams(4, 2, "actor", device="cpu")
    deep = NetParams(4, 2, "actor", device="cpu", n_layers=2)
    other_ed = NetParams(2, 2, "actor", device="cpu")
    assert check_nets([a, a.clone()], 2)[1].edge_dim == 4
    assert check_nets(a, 1) == [a]
    with pytest.raises(ValueError, match="n_layers"):
        check_nets([a, deep], 2)
    with pytest.raises(ValueError, match="edge_dim"):
        check_nets([a, other_ed], 2)
    with pytest.raises(ValueError, match="runs 3 networks, got 2"):
        check_nets([a, a], 3)


# ------------------------------------------------------------------ test.py --all-steps / --paths
def _test_cli():
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_sweep", os.path.join(ROOT, "test.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, lambda argv: mod.build_test_parser().parse_args(argv + ["--area-size", "2.0"])


def _run_dir(root, name, steps=(), **config):
    import train
    run = os.path.join(root, name)
    os.makedirs(os.path.join(run, "models"))
    for s in steps:
        os.makedirs(os.path.join(run, "models", str(s)))
    base = dict(env="DoubleIntegrator", num_agents=8, gnn_layers=1, n_rays=32, algo="gcbf+")
    base.update(config)
    train.write_config(run, argparse.Namespace(**base), {"alpha": 1.0})
    return run


def test_sweep_flag_parsing_and_refusals():
    cli, parse = _test_cli()
    args = parse(["--paths", "a", "b", "--all-steps"])
    assert args.paths == ["a", "b"] and args.all_steps and cli.check_sweep_flags(args)
    assert cli.check_sweep_flags(parse(["--path", "a", "--all-steps"]))
    assert cli.check_sweep_flags(parse(["--paths", "a", "--step", "3"]))
    assert not cli.check_sweep_flags(parse(["--path", "a"]))
    for argv, what in ((["--paths", "a", "--path", "b"], "mutually exclusive"),
                       (["--all-steps"], "--path"),
                       (["--path", "a", "--all-steps", "--step", "2"], "--step"),
                       (["--path", "a", "--all-steps", "--u-ref"], "--u-ref"),
                       (["--paths", "a", "--online-refine"], "--online-refine"),
                       (["--path", "a", "--all-steps", "--qp-filter"], "--qp-filter"),
                       (["--paths", "a", "b", "--cbf", "0"], "--cbf"),
                       (["--path", "a", "--all-steps", "--algo", "dec_share_cbf"], "dec_share_cbf"),
                       (["--paths", "a", "--algo", "centralized_cbf"], "centralized_cbf")):
        with pytest.raises(SystemExit, match=what):
            cli.check_sweep_flags(parse(argv))
        with pytest.raises(SystemExit, match=what):   # refused before any run directory is read
            cli.test(parse(argv))


def test_all_steps_finds_and_sorts_checkpoints(tmp_path):
    cli, parse = _test_cli()
    run = _run_dir(str(tmp_path), "run", steps=(100, 2, 10))
    os.makedirs(os.path.join(run, "models", "tmp"))
    assert cli.checkpoint_steps(run) == [2, 10, 100]
    assert cli.sweep_networks(parse(["--path", run, "--all-steps"]), [run]) == [(run, 2), (run, 10), (run, 100)]
    other = _run_dir(str(tmp_path), "other", steps=(5, 7))
    args = parse(["--paths", run, other])
    assert cli.sweep_networks(args, [run, other]) == [(run, 100), (other, 7)]
    args = parse(["--paths", run, other, "--step", "5"])
    assert cli.sweep_networks(args, [run, other]) == [(run, 5), (other, 5)]
    empty = _run_dir(str(tmp_path), "empty")
    with pytest.raises(SystemExit, match="no checkpoints"):
        cli.checkpoint_steps(empty)


@pytest.mark.parametrize("key,value", [("env", "SingleIntegrator"), ("num_agents", 16), ("gnn_layers", 2),
                                       ("n_rays", 16)])
def test_paths_refuse_runs_of_another_configuration(tmp_path, key, value):
    cli, parse = _test_cli()
    a = _run_dir(str(tmp_path), "a", steps=(1,))
    b = _run_dir(str(tmp_path), "b", steps=(1,), **{key: value})
    configs = [cli.read_config(a), cli.read_config(b)]
    cli.check_sweep_configs([a, a], [configs[0], configs[0]])
    with pytest.raises(SystemExit, match=f"{key} = "):
        cli.check_sweep_configs([a, b], configs)
    with pytest.raises(SystemExit, match=key):
        cli.test(parse(["--paths", a, b]))
