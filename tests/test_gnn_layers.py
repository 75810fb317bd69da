"""CPU: networks with more than one GNN layer (gnn.py:78-104, n_layers = --gnn-layers): parameter names, shapes and
counts, the library's flat layout, checkpoints in the reference pickle layout, and the multi-layer oracle."""
import numpy as np
import pytest
import torch

from gnn_layers_oracle import init_params, layer_specs as oracle_specs, net_forward
from helpers import oracle_env, random_scene

# parameters added by every layer after the first: msg (ed + 256) x 256, the rest as layer 0, update/Dense_0 256 x 256
EXTRA = {2: 362625, 4: 363137, 6: 363649}
L2_COUNTS = {"SingleIntegrator": (2, 2, 728323, 728580), "DoubleIntegrator": (4, 2, 729347, 729604),
             "LinearDrone": (6, 3, 730371, 730885)}


def test_specs_names_shapes_and_counts():
    from gcbfplus_b200.algo.params import layer_specs
    for env_id, (ed, nu, cbf2, act2) in L2_COUNTS.items():
        assert sum(i * o + o for _, i, o in layer_specs(ed, 1, "cbf", 2)) == cbf2, env_id
        assert sum(i * o + o for _, i, o in layer_specs(ed, nu, "actor", 2)) == act2, env_id
        for L in (2, 3):
            n1 = sum(i * o + o for _, i, o in layer_specs(ed, nu, "actor"))
            assert sum(i * o + o for _, i, o in layer_specs(ed, nu, "actor", L)) == n1 + (L - 1) * EXTRA[ed]
        specs = layer_specs(ed, nu, "actor", 3)
        assert specs == oracle_specs(ed, nu, "actor", 3)
        assert specs[:9] == layer_specs(ed, nu, "actor")[:9] and specs[-3:] == layer_specs(ed, nu, "actor")[-3:]
        for l in (1, 2):
            layer = dict((p.split("/", 3)[3], (i, o)) for p, i, o in specs[9 * l: 9 * l + 9])
            assert all(p.startswith(f"params/GNN_0/GNNLayer_{l}/") for p, _, _ in specs[9 * l: 9 * l + 9])
            assert layer["msg/Dense_0"] == (ed + 256, 256) and layer["update/Dense_0"] == (256, 256)
            assert layer["Dense_0"] == (256, 128) and layer["Dense_2"] == (256, 128) and layer["Dense_1"] == (128, 1)


# the tf32 planes of the GEMM weights (gcbf_params_t_count_l): hi and lo of the transposed weights of every layer and, at
# L = 1, of the straight ones the backward reads.  The 9 GEMM weights of a layer hold 360448 floats at any ed
# (layer 0: update/Dense_0 rows 3..130 and the two hidden head layers; later layers: Ws and Wr instead).
PLANE_FLOATS = {1: 4 * 360448, 2: 2 * 2 * 360448, 3: 2 * 3 * 360448}


@pytest.mark.parametrize("L", [1, 2, 3])
@pytest.mark.parametrize("ed,nu", [(2, 2), (4, 2), (6, 3)])
def test_library_layout_and_planes_follow_the_specs(ed, nu, L):
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo.params import layer_specs
    lib = _lib.load()
    specs = layer_specs(ed, nu, "actor", L)
    offs = _lib.param_offsets(ed, nu, L)
    assert len(offs) == 2 * len(specs) == 2 * (9 * L + 3)
    assert all(o % 4 == 0 for o in offs) and offs == sorted(offs)
    ends = offs[1:] + [_lib.param_count(ed, nu, L)]
    for k, (_, fi, fo) in enumerate(specs):
        assert ends[2 * k] - offs[2 * k] >= fi * fo and ends[2 * k] - offs[2 * k] < fi * fo + 4
        assert ends[2 * k + 1] - offs[2 * k + 1] >= fo
    assert lib.gcbf_params_t_count_l(ed, nu, L) == PLANE_FLOATS[L]
    assert lib.gcbf_param_count_l(ed, nu, 0) < 0 and lib.gcbf_param_count_l(ed, nu, 9) < 0
    assert lib.gcbf_params_t_count_l(ed, nu, 0) < 0 and lib.gcbf_params_t_count_l(ed, nu, 9) < 0


@pytest.mark.parametrize("L", [2, 3])
def test_checkpoint_round_trip_in_reference_layout(tmp_path, L):
    from gcbfplus_b200.algo.params import NetParams, flatten_tree, load_pickle
    p = NetParams(4, 2, "actor", device="cpu", n_layers=L).init_xavier(7)
    path = str(tmp_path / "actor.pkl")
    p.save(path)
    tree = load_pickle(path)
    flat = flatten_tree(tree)
    assert sorted(flat) == sorted(k for s, _, _ in p.specs for k in (s + "/kernel", s + "/bias"))
    assert flat[f"params/GNN_0/GNNLayer_{L - 1}/msg/Dense_0/kernel"].shape == (4 + 256, 256)
    # same xavier stream as the oracle's init
    ref = flatten_tree(init_params(4, 2, "actor", 7, L))
    for k, v in ref.items():
        np.testing.assert_array_equal(flat[k], v)
    q = NetParams(4, 2, "actor", device="cpu", n_layers=L).load(path)
    assert torch.equal(q.flat, p.flat)
    assert q.clone().n_layers == L
    with pytest.raises(KeyError):   # a deeper network does not load a shallower checkpoint
        NetParams(4, 2, "actor", device="cpu", n_layers=L + 1).load(path)
    for shallower in range(1, L):   # nor a shallower network a deeper checkpoint's first layers only
        with pytest.raises(ValueError, match=f"GNNLayer_{shallower}"):
            NetParams(4, 2, "actor", device="cpu", n_layers=shallower).load(path)


def test_train_py_rejects_deep_networks_before_any_work(tmp_path):
    """train.py --gnn-layers 2 stops before it creates a device, a log directory or a run (the train step implements
    one GNN layer); Trainer rejects such a network at construction."""
    import train
    from gcbfplus_b200.algo.train import require_one_layer
    log_dir = tmp_path / "logs"
    args = train.build_parser(train.FLAGS).parse_args(["--env", "DoubleIntegrator", "-n", "4", "--area-size", "2",
                                                      "--gnn-layers", "2", "--log-dir", str(log_dir)])
    with pytest.raises(NotImplementedError, match="gnn_layers = 1"):
        train.train(args)
    assert not log_dir.exists()
    require_one_layer(1, "training")


def _to_torch(tree, dtype):
    from oracle.nn import to_torch
    return to_torch(tree, dtype)


@pytest.mark.parametrize("env_id", ["DoubleIntegrator", "LinearDrone"])
def test_oracle_dense_equals_sparse_at_two_layers(env_id):
    """The dense reference layout (masked edges to the pad node, every node row computed) and the sparse edge set the
    CUDA path uses give the same h and pi at L = 2: goal / hit / pad rows never reach an agent except as senders."""
    N, area, n_obs = 8, 1.5, 4
    agent, goal, obs = random_scene(env_id, N, 1, area, n_obs, seed=5)
    oenv = oracle_env(env_id, N, area, n_obs, dtype=torch.float64)
    nu = 3 if env_id == "LinearDrone" else 2
    ed = oenv.state_dim
    cp = _to_torch(init_params(ed, 1, "cbf", 1, 2), torch.float64)
    ap = _to_torch(init_params(ed, nu, "actor", 2, 2), torch.float64)
    dense = oenv.get_graph(torch.from_numpy(agent[0]).double(), torch.from_numpy(goal[0]).double(),
                           _obstacles64(obs, env_id))
    sparse = oenv.sparsify(dense)
    assert sparse.receivers.numel() < dense.receivers.numel()
    assert (sparse.senders >= 2 * N).any()      # hit senders present: their constant rows are exercised
    with torch.no_grad():
        for p, kind in ((cp, "cbf"), (ap, "actor")):
            a, b = net_forward(p, dense, kind), net_forward(p, sparse, kind)
            np.testing.assert_allclose(a.numpy(), b.numpy(), rtol=0, atol=1e-12)


def _obstacles64(obs, env_id):
    from oracle.geometry import Rectangle, Sphere
    if "radius" in obs:
        return Sphere.create(obs["center"][0], obs["radius"][0], dtype=torch.float64)
    return Rectangle.create(obs["center"][0], obs["width"][0], obs["height"][0], obs["theta"][0], dtype=torch.float64)


def _chain_jacobian(L):
    """dh/dx of the CBF over a chain of agents spaced 0.4 apart (comm radius 0.5: each agent sees only its chain
    neighbours), no obstacles, edge features through add_edge_feats as in the QP (gcbf_plus.py:310-320)."""
    N = 6
    oenv = oracle_env("DoubleIntegrator", N, 4.0, 0, dtype=torch.float64)
    agent = torch.zeros(N, 4, dtype=torch.float64)
    agent[:, 0] = 0.5 + 0.4 * torch.arange(N, dtype=torch.float64)
    agent[:, 1] = 1.0 + 0.01 * torch.arange(N, dtype=torch.float64) ** 2
    agent[:, 2:] = 0.1 * torch.sin(torch.arange(2 * N, dtype=torch.float64)).reshape(N, 2)
    goal = agent.clone()
    goal[:, 1] += 1.0
    g = oenv.sparsify(oenv.get_graph(agent, goal, None))
    cp = _to_torch(init_params(4, 1, "cbf", 3, L), torch.float64)
    rest = g.states[N:]

    def h_aug(x):
        return net_forward(cp, oenv.add_edge_feats(g, torch.cat([x, rest[: g.states.shape[0] - N]], 0)), "cbf")[:, 0]

    J = torch.autograd.functional.jacobian(h_aug, agent.clone())      # [N, N, sd]
    adj = np.eye(N, dtype=int)
    for r, s in zip(g.receivers.tolist(), g.senders.tolist()):
        if s < N:
            adj[r, s] = 1
    return J.abs().sum(-1).numpy(), adj


def test_oracle_jacobian_is_nonzero_exactly_on_the_two_hop_ball():
    J1, adj = _chain_jacobian(1)
    J2, _ = _chain_jacobian(2)
    two_hop = (adj @ adj) > 0
    assert ((J1 > 0) == (adj > 0)).all()
    assert ((J2 > 0) == two_hop).all()
    assert (two_hop & ~(adj > 0)).any()      # the chain has pairs two hops apart that one layer does not couple
