"""CPU: the NumPy replica of the rollout noise (tests/noise_oracle.py) against numpy.random.Philox and the normal
distribution, Perturbation's validation, and test.py's noise flag handling."""
import importlib.util
import os
import sys

import numpy as np
import pytest

import noise_oracle as no
from helpers import ROOT


@pytest.mark.parametrize("counter,key", [((0, 0, 0, 0), (0, 0)), ((5, 7, 11, 3), (1234, 2)),
                                         ((2 ** 62 + 5, 2 ** 63 - 1, 12345678901234, 9), (2 ** 64 - 3, 1)),
                                         ((255, 3, 511, 1), (2 ** 63 + 17, 2)),
                                         ((2 ** 64 - 1, 5, 1, 0), (3, 0))])   # the pre-increment carries into word 1
def test_philox_replica_equals_numpy_philox(counter, key):
    gen = np.random.Philox(counter=np.array(counter, dtype=np.uint64), key=np.array(key, dtype=np.uint64))
    want = gen.random_raw(8)
    c = np.array([counter, counter], dtype=np.uint64)
    with np.errstate(over="ignore"):
        for k in range(2):                      # numpy increments the 256-bit counter before each block
            for _ in range(k + 1):
                c[k, 0] += np.uint64(1)
                if c[k, 0] == 0:
                    c[k, 1] += np.uint64(1)
    got = no.philox(c, key).reshape(-1)
    assert np.array_equal(got, want)


def test_box_muller_draws_are_standard_normal():
    rng = np.random.default_rng(3)
    c = rng.integers(0, 2 ** 63, size=(250_000, 4), dtype=np.uint64)
    z = no.normals(1234, no.STATE, c).astype(np.float64).ravel()
    n = z.size
    assert n == 10 ** 6
    se_mean = 1.0 / np.sqrt(n)
    se_var = np.sqrt(2.0 / n)               # standard error of the sample variance of N(0, 1)
    assert abs(z.mean()) < 4 * se_mean, z.mean()
    assert abs(z.var() - 1.0) < 4 * se_var, z.var()
    # the pairs of one call are independent (z0 and z1 share u0): no correlation within four standard errors
    zz = z.reshape(-1, 4)
    assert abs(np.mean(zz[:, 0] * zz[:, 1])) < 4 / np.sqrt(zz.shape[0])


def test_component_layout_and_zero_sigma():
    """Block j of an agent covers its components 4j .. 4j + 3; sigma 0 copies (-0.0 included); draws of one episode do
    not depend on the other episodes of the batch."""
    z = no.component_z(7, no.LIDAR, 3, [4, 9], 5, 64)
    for e, env in enumerate((4, 9)):
        for i in range(5):
            for j in range(16):
                want = no.normals(7, no.LIDAR, np.array([[3, env, i, j]], dtype=np.uint64))[0]
                assert np.array_equal(z[e, i, 4 * j:4 * j + 4], want)
    assert np.array_equal(no.component_z(7, no.LIDAR, 3, [9], 5, 64)[0], z[1])
    x = np.array([[[-0.0, 1.5, 2.0, -3.0]]], dtype=np.float32)
    out = no.perturb(x, [0.0, 0.0, 0.0, 0.0], np.ones((1, 1, 4), dtype=np.float32))
    assert out.tobytes() == x.tobytes()


def test_perturbation_validation():
    from gcbfplus_b200.trainer.rollout import Perturbation

    class Env:
        state_dim, action_dim = 4, 2
    p = Perturbation(0.1, 0.02, [0.1, 0.2], seed=5, env_offset=3)
    assert p.sigmas(Env) == ([0.1] * 4, 0.02, [0.1, 0.2])
    assert Perturbation([0.1, 0.2, 0.3, 0.4], 0.0, 0.0, seed=0).sigmas(Env)[0] == [0.1, 0.2, 0.3, 0.4]
    buf = Perturbation([0.1, 0.2, 0.3, 0.4], 0.5, [0.6, 0.7], seed=2 ** 64 - 1).pack(Env).numpy()
    assert buf.view(np.uint64)[0] == 2 ** 64 - 1
    assert np.array_equal(buf[2:6], np.float32([0.1, 0.2, 0.3, 0.4])) and buf[8] == np.float32(0.5)
    assert np.array_equal(buf[9:11], np.float32([0.6, 0.7])) and not buf[6:8].any() and not buf[11:].any()
    with pytest.raises(ValueError, match="state_sigma has 3 values"):
        Perturbation([0.1, 0.2, 0.3], 0.0, 0.0, seed=0).sigmas(Env)
    with pytest.raises(ValueError, match="action_sigma has 3 values"):
        Perturbation(0.1, 0.0, [0.1, 0.1, 0.1], seed=0).sigmas(Env)
    for kw, what in ((dict(state_sigma=-0.1), "state_sigma must be finite and >= 0"),
                     (dict(lidar_sigma=float("nan")), "lidar_sigma must be finite"),
                     (dict(action_sigma=[0.1, float("inf")]), "action_sigma must be finite"),
                     (dict(lidar_sigma=[0.1, 0.2]), "lidar_sigma is one value"),
                     (dict(state_sigma=[]), "state_sigma is empty"),
                     (dict(seed=-1), "seed"), (dict(seed=2 ** 64), "seed"), (dict(seed=1.5), "seed"),
                     (dict(env_offset=-2), "env_offset")):
        args = dict(state_sigma=0.1, lidar_sigma=0.0, action_sigma=0.0, seed=0)
        args.update(kw)
        with pytest.raises(ValueError, match=what):
            Perturbation(**args)


def test_engine_refuses_persistent_and_several_networks_with_a_perturbation():
    """Checked before any buffer is allocated (the environment is never touched)."""
    from gcbfplus_b200.trainer.rollout import Perturbation, RolloutEngine

    class Env:
        params = {"n_obs": 0}
        max_episode_steps = 4
        device = "cpu"
        enable_stop = True
    p = Perturbation(0.1, 0.0, 0.0, seed=0)
    with pytest.raises(ValueError, match="persistent rollout has no noise model"):
        RolloutEngine(Env, 2, persistent=True, perturbation=p)
    with pytest.raises(ValueError, match="n_nets = 1"):
        RolloutEngine(Env, 2, n_nets=2, perturbation=p)


def _test_cli():
    sys.path.insert(0, ROOT)
    spec = importlib.util.spec_from_file_location("gcbf_test_cli_noise", os.path.join(ROOT, "test.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod, lambda argv: mod.build_test_parser().parse_args(argv)


def test_noise_flag_parsing_and_rejections():
    cli, parse = _test_cli()
    a = parse(["--path", "runs/x", "--area-size", "4", "--state-noise", "0.1", "0.2", "0.1", "0.2", "--lidar-noise",
               "0.02", "--action-noise", "0.1", "--offset", "3"])
    p = cli.noise_perturbation(a)
    assert p.state_sigma == (0.1, 0.2, 0.1, 0.2) and p.lidar_sigma == 0.02 and p.action_sigma == (0.1,)
    assert p.seed == a.seed == 1234 and p.env_offset == 3
    assert cli.noise_perturbation(parse(["--path", "r", "--area-size", "4", "--lidar-noise", "0.1",
                                         "--noise-seed", "9"])).seed == 9
    assert cli.noise_perturbation(parse(["--path", "r", "--area-size", "4"])) is None
    for argv, what in ((["--paths", "runs/a", "runs/b", "--state-noise", "0.1"], "--state-noise .* --paths"),
                       (["--path", "runs/a", "--all-steps", "--lidar-noise", "0.1"], "--lidar-noise .* --all-steps"),
                       (["--path", "runs/a", "--falsify", "5", "--action-noise", "0.1"], "--action-noise .* --falsify"),
                       (["--path", "runs/a", "--noise-seed", "3"], "--noise-seed"),
                       (["--path", "runs/a", "--state-noise", "-0.1"], "state_sigma must be finite and >= 0")):
        argv = argv + ["--area-size", "2.0"]
        with pytest.raises(SystemExit, match=what):
            cli.noise_perturbation(parse(argv))
        # refused before anything is built or loaded (the run directories do not exist)
        with pytest.raises(SystemExit, match=what):
            cli.test(parse(argv))
