"""CPU: the CBF-QP baseline entry points are exported, reject bad arguments before enqueueing anything, and the
Python surface matches the reference's (make_algo names, methods that raise)."""
import ctypes

import pytest

CBFQP_SYMBOLS = ("gcbf_cbf_pairwise", "gcbf_cbfqp_workspace_floats", "gcbf_cbfqp_dec_share", "gcbf_cbfqp_centralized")


def test_cbfqp_symbols_exported():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    for n in CBFQP_SYMBOLS:
        assert hasattr(lib, n), n
        assert n in _lib._SIGNATURES, n


def _desc(kind=1, G=2, N=8, R=32):
    from gcbfplus_b200 import _lib
    d = _lib.EnvDesc()
    d.env_kind, d.n_graphs, d.n_agents, d.n_hits = kind, G, N, R
    d.u_lim = 1.0
    return d


def test_cbfqp_argument_errors_without_gpu():
    from gcbfplus_b200 import _lib
    lib = _lib.load()
    d = _desc()
    n = lib.gcbf_cbfqp_workspace_floats(ctypes.byref(d))
    assert n >= 2 * 8 * 3 * (3 + 2 * 2)
    p = ctypes.c_void_p(16)   # never dereferenced: every call below fails its argument checks first
    rc = lib.gcbf_cbfqp_dec_share(ctypes.byref(d), 1.0, 0, 1e-7, p, p, p, p, None, None, p, n, None)
    assert rc < 0 and b"max_iter" in lib.gcbf_last_error_string()
    rc = lib.gcbf_cbfqp_dec_share(ctypes.byref(d), 1.0, 10, 1e-7, p, p, p, p, None, None, p, n - 1, None)
    assert rc < 0 and b"workspace" in lib.gcbf_last_error_string()
    big = _desc(N=1025)
    nb = lib.gcbf_cbfqp_workspace_floats(ctypes.byref(big))
    rc = lib.gcbf_cbfqp_centralized(ctypes.byref(big), 1.0, 10, 1e-7, p, p, p, p, None, None, p, nb, None)
    assert rc < 0 and b"1024" in lib.gcbf_last_error_string()
    # LinearDrone (NU = 3): 999 agents take 232,284 B of shared memory, 1000 would take 232,516 > 227 KB
    drone = _desc(kind=3, N=1000)
    nd = lib.gcbf_cbfqp_workspace_floats(ctypes.byref(drone))
    rc = lib.gcbf_cbfqp_centralized(ctypes.byref(drone), 1.0, 10, 1e-7, p, p, p, p, None, None, p, nd, None)
    msg = lib.gcbf_last_error_string()
    assert rc < 0 and b"1000 agents" in msg and b"LinearDrone 999" in msg, msg
    tiny = _desc(N=1, R=1)
    rc = lib.gcbf_cbf_pairwise(ctypes.byref(tiny), p, p, p, p, p, p, p, None, None)
    assert rc < 0 and b"candidates" in lib.gcbf_last_error_string()
    d.n_rays, d.edge_cap = 32, 64
    rc = lib.gcbf_env_step(ctypes.byref(d), p, p, None, None, p, p, p, p, p, p, p, 4, None)
    assert rc < 0 and b"mode" in lib.gcbf_last_error_string()


def test_make_algo_baselines_surface():
    from gcbfplus_b200.algo import CentralizedCBF, DecShareCBF, make_algo
    from gcbfplus_b200.env import make_env
    env = make_env("DubinsCar", 4, area_size=2.0, num_obs=0, device="cpu")
    kw = dict(env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
              action_dim=env.action_dim, n_agents=env.num_agents, alpha=2.0)
    c = make_algo("centralized_cbf", **kw)
    assert isinstance(c, CentralizedCBF) and c.config == {"alpha": 2.0} and env.enable_stop
    d = make_algo("dec_share_cbf", **kw)
    assert isinstance(d, DecShareCBF) and not env.enable_stop and env.action_step_mode == 3
    for algo in (c, d):
        with pytest.raises(NotImplementedError):
            algo.actor_params
        for call in (lambda: algo.step(None, None), lambda: algo.update(None, 0), lambda: algo.save("x", 0),
                     lambda: algo.load("x", 0)):
            with pytest.raises(NotImplementedError):
                call()
    with pytest.raises(NotImplementedError):
        make_algo("gcbf", **kw)
