"""GPU: every GNN forward path against float64 (tests/gnn_f64.py): |got - f64| <= C_BAR * unit per output tensor
(C_BAR_TC on the 3xTF32 tensor-core path), where the unit is the size of fp32 rounding of the case
(tests/test_gnn_f64_cpu.py shows the bar accepts the float32 oracle and rejects a dropped edge or a message / update /
head layer at tf32 precision).

A. gcbf_gnn_infer (the folded rollout network) and gcbf_gnn_forward_l at 1-3 layers, called through the C ABI on crafted
   graphs: a degree ladder 1 .. 64 (across the rd <= 4 fast path), a >= 300-row receiver straddling 4 edge tiles, edge
   counts around the 128-row tile, more than 4 tiles per CTA, node rows around 128, slack rows past the edge counter
   holding valid but wrong indices, goal / agent / hit senders, clip_all 0 and 1.
B. Softmax edges: gate bias at +-90, a gate kernel scaled by 50, tied logits.
C. Rollout records (5-launch step path, persistent kernel, several networks in one launch): every recorded action of
   the sampled environments against the float64 2 pi + u_ref of the graph rebuilt from the recorded state.
D. Every GEMM of gcbf_gnn_forward_l (one layer) against float64 of its own saved input, in units of
   2^-24 (|x| |W| + |b|): the bar that catches a GEMM at the wrong precision on the tensor-core path.
Run with -s to see max err / unit of every case."""
import ctypes as C

import numpy as np
import pytest
import torch

import gnn_f64 as F
from helpers import oracle_env, product_algo, product_env, product_obstacles, random_scene

pytestmark = pytest.mark.gpu

WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    print("\nmax err / unit per path:")
    for k in sorted(WORST):
        print(f"  {k:34s} {WORST[k]:7.2f}")


def _note(path, r, what):
    WORST[path] = max(WORST.get(path, 0.0), r)
    print(f"{path:24s} {what:52s} err/unit {r:7.2f}")


def _net(env, kind, L, seed=None, env_id=None):
    """Pretrained fixture (L = 1, seed None) or a xavier network with L GNN layers."""
    from gcbfplus_b200.algo.params import NetParams
    if seed is None:
        algo = product_algo(env, env_id)
        return algo.actor_params if kind == "actor" else algo.cbf_params
    return NetParams(env.edge_dim, env.action_dim if kind == "actor" else 1, kind, n_layers=L).init_xavier(seed)


def _variant(net, name):
    """A copy of `net` with one of F.softmax_variants applied."""
    from gcbfplus_b200.algo.params import NetParams
    p = F.softmax_variants({k: torch.from_numpy(np.asarray(v)) for k, v in _flat(net.to_tree()).items()})[name]
    out = NetParams(net.edge_dim, net.out_dim, net.kind, n_layers=net.n_layers)
    from gcbfplus_b200.algo.params import unflatten_tree
    return out.from_tree(unflatten_tree({k: v.numpy() for k, v in p.items()}))


def _flat(tree):
    from gcbfplus_b200.algo.params import flatten_tree
    return flatten_tree(tree)


def _run(env, net, entry, arrays, clip_all):
    """One C ABI forward on device arrays (agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters)."""
    from gcbfplus_b200 import _lib
    agent, edge_recv = arrays[0], arrays[5]
    G, N = agent.shape[:2]
    d = env.desc(G, 0, edge_cap=edge_recv.numel())
    kind = _lib.NET_CBF if net.kind == "cbf" else _lib.NET_ACTOR
    out = torch.full((G, N, net.out_dim), float("nan"), device="cuda")
    ws = torch.empty(int(env.lib.gcbf_gnn_workspace_floats_l(C.byref(d), net.out_dim, net.n_layers)), device="cuda")
    st = torch.cuda.current_stream().cuda_stream
    ptrs = [_lib.ptr(a) for a in arrays]
    if entry == "infer":
        blob = torch.zeros(int(env.lib.gcbf_infer_count(env.edge_dim, net.out_dim)), device="cuda")
        _lib.check(env.lib.gcbf_prepare_infer(env.edge_dim, net.out_dim, _lib.ptr(net.flat), _lib.ptr(blob), st),
                   "gcbf_prepare_infer")
        rc = env.lib.gcbf_gnn_infer(C.byref(d), kind, net.out_dim, _lib.ptr(net.flat), _lib.ptr(blob),
                                    1 if _lib.USE_TC else 0, *ptrs, clip_all, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
                                    st)
    else:
        rc = env.lib.gcbf_gnn_forward_l(C.byref(d), kind, net.out_dim, net.n_layers, _lib.ptr(net.flat),
                                        _lib.ptr(net.prepared(st)), *ptrs, clip_all, _lib.ptr(out), _lib.ptr(ws),
                                        ws.numel(), st)
    _lib.check(rc, entry)
    torch.cuda.synchronize()
    return out.cpu()


def _device(agent, goal, hits, lists):
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    return [t(agent), t(goal), t(hits)] + [t(a) for a in lists]


def _check(env_id, env, arrays, clip_all, graphs, what, gemm_path, nets):
    """Run every (entry, net) of `nets` and compare graphs `graphs` with float64."""
    N = arrays[0].shape[1]
    oenv = oracle_env(env_id, N, 2.0, 0, dtype=torch.float64)
    host = [a.cpu() for a in arrays]
    ogs = {g: F.oracle_graph(oenv, *host, clip_all, g) for g in graphs}
    for entry, net in nets:
        if (entry != "infer" and net.n_layers > 1) and gemm_path != "tc":
            continue
        got = _run(env, net, entry, arrays, clip_all)
        p = F.params64(net)
        worst = 0.0
        for g, og in ogs.items():
            ref = F.forward(p, og, net.kind)
            worst = max(worst, F.ratio(got[g], ref, F.unit(p, og, net.kind, ref)))
        path = f"{entry} L={net.n_layers} {gemm_path}" if entry != "infer" else f"infer {gemm_path}"
        _note(path, worst, f"{env_id} {what} {net.kind} clip{clip_all}")
        assert worst <= (F.C_BAR_TC if gemm_path == "tc" else F.C_BAR), (entry, net.kind, net.n_layers, what, worst)


def _nets(env, env_id, deep=True):
    out = [("infer", _net(env, "actor", 1, env_id=env_id)), ("infer", _net(env, "cbf", 1, env_id=env_id)),
           ("forward_l", _net(env, "actor", 1, env_id=env_id)), ("forward_l", _net(env, "cbf", 1, env_id=env_id))]
    if deep:
        out += [("forward_l", _net(env, "actor", 2, seed=5)), ("forward_l", _net(env, "cbf", 3, seed=6))]
    return out


def _synthetic(env_id, N, G, codes, seed=3, slack=37, order=None):
    agent, goal, hits = F.synthetic_scene(env_id, N, G, 2.0, seed)
    lists = F.write_rows(codes, N, order=order, cap=sum(map(len, codes)) + slack)
    return _device(agent, goal, hits, lists)


def _R(env_id):
    return 16 if env_id in ("DubinsCar", "LinearDrone") else 32


ENVS = ["SingleIntegrator", "DoubleIntegrator", "DubinsCar", "LinearDrone"]


# ------------------------------------------------------------------ A. crafted graphs
@pytest.mark.parametrize("env_id", ENVS)
def test_degree_ladder(env_id, gemm_path):
    """Receivers of degree 1 .. 64 in three graphs, rows in reverse receiver order, slack rows past the counter."""
    N, area, seed = F.LADDER_SCENE
    env = product_env(env_id, N, area, 0)
    codes = F.ladder_codes(N, _R(env_id), G=3)
    arrays = _synthetic(env_id, N, 3, codes, seed, order=range(3 * N - 1, -1, -1))
    for clip_all in (0, 1):
        _check(env_id, env, arrays, clip_all, [0, 1, 2], "ladder", gemm_path, _nets(env, env_id))


@pytest.mark.parametrize("env_id", ENVS)
def test_hub_straddles_edge_tiles(env_id, gemm_path):
    """A receiver with N + R >= 336 rows (goal, every other agent, every hit) starting 3 rows before the 128-row
    boundary: rows 125 .. 125 + N + R cross 3 boundaries."""
    N = 320
    env = product_env(env_id, N, 2.0, 0)
    codes = F.ladder_codes(N, _R(env_id), degrees=(5,) * 25 + (N + _R(env_id),))
    arrays = _synthetic(env_id, N, 1, codes)
    assert int(arrays[3][25]) == 125 and int(arrays[4][25]) >= 300
    _check(env_id, env, arrays, 0, [0], "hub", gemm_path, _nets(env, env_id))


@pytest.mark.parametrize("env_id", ["DoubleIntegrator", "LinearDrone"])
def test_edge_count_ladder(env_id, gemm_path):
    """Edge counters 1, 127, 128, 129, 255, 256, 257: the last tile full, one row short or one row over."""
    N = 64
    env = product_env(env_id, N, 2.0, 0)
    for n in (1, 127, 128, 129, 255, 256, 257):
        degrees = [min(5, max(n - 5 * i, 0)) for i in range(N)]
        assert sum(degrees) == n
        arrays = _synthetic(env_id, N, 1, F.ladder_codes(N, _R(env_id), degrees=degrees))
        _check(env_id, env, arrays, 0, [0], f"{n} edges", gemm_path, _nets(env, env_id, deep=n in (128, 129)))


def test_more_than_four_tiles_per_cta(gemm_path):
    """9 x 512 agents with 12-20 rows each: more than 4 * SMs * 128 rows (67584 on a 132-SM H100), so every CTA of the
    edge kernels loops over more than 4 tiles; the last graph holds the rows beyond that."""
    env_id, N, G = "DoubleIntegrator", 512, 9
    env = product_env(env_id, N, 2.0, 0)
    rng = np.random.Generator(np.random.PCG64(8))
    codes = F.ladder_codes(N, 32, G=G, degrees=rng.integers(12, 21, size=N).tolist())
    arrays = _synthetic(env_id, N, G, codes, seed=9)
    rows = 4 * torch.cuda.get_device_properties(0).multi_processor_count * 128
    assert int(arrays[7][0]) > rows and int(arrays[3][(G - 1) * N]) < rows
    _check(env_id, env, arrays, 0, [0, G - 1], "9x512 many tiles", gemm_path, _nets(env, env_id, deep=False))


@pytest.mark.parametrize("N,G", [(1, 1), (127, 1), (128, 1), (129, 1), (1, 3), (43, 3), (126, 1)])
def test_node_rows(N, G, gemm_path):
    """A = G N node rows around the 128-row GEMM tile (L > 1: A + 2 rows, crossing it at N = 126 and 127)."""
    env_id = "DoubleIntegrator"
    env = product_env(env_id, N, 2.0, 0)
    arrays = _synthetic(env_id, N, G, F.ladder_codes(N, 32, G=G, degrees=()))
    _check(env_id, env, arrays, 0, sorted({0, G - 1}), f"A={N * G}", gemm_path, _nets(env, env_id))


def _crafted_scene(env_id, seed=2):
    """A dense cluster (hub), isolated agents and rings of 12 with exactly two neighbours each, among obstacles."""
    N = 64
    rng = np.random.Generator(np.random.PCG64(seed))
    agent, goal, obs = random_scene(env_id, N, 1, 4.0, 6, seed)
    pd = 3 if env_id == "LinearDrone" else 2
    pos = np.zeros((N, pd))
    pos[:20, :2] = 1.0 + rng.uniform(-0.2, 0.2, size=(20, 2))
    pos[20:28, :2] = np.stack([np.arange(8) * 1.5 + 0.5, np.full(8, 8.0)], 1)
    for r in range(3):
        th = 2 * np.pi * np.arange(12) / 12 + 0.1 * r
        pos[28 + 12 * r:40 + 12 * r, :2] = np.stack([2.5 + 2.2 * r + 0.773 * np.cos(th), 2.5 + 0.773 * np.sin(th)], 1)
    if pd == 3:
        pos[:, 2] = 1.0 + rng.uniform(-0.05, 0.05, size=N)
    agent[0, :, :pd] = pos
    obs["center"][0, 0, :2] = 1.25            # an obstacle next to the cluster: active hit senders
    return agent, goal, obs


@pytest.mark.parametrize("env_id", ENVS)
def test_real_graphs(env_id, gemm_path):
    """env.get_graph's own lists (canonical rows) of a crafted scene, with active hits."""
    agent, goal, obs = _crafted_scene(env_id)
    N = agent.shape[1]
    env = product_env(env_id, N, 4.0, 6)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(),
                          product_obstacles(env_id, obs), edge_cap=N * (N + env.n_hits))
    torch.cuda.synchronize()
    graph.check_overflow()
    rd = graph.row_deg.cpu()
    assert int(rd.max()) >= 20 and int((rd == 1).sum()) >= 4 and int((graph.edge_src < -1).sum()) > 0
    arrays = [graph.agent, graph.goal, graph.hits, graph.row_start, graph.row_deg, graph.edge_recv, graph.edge_src,
              graph.counters]
    for clip_all in (0, 1):
        _check(env_id, env, arrays, clip_all, [0], "crafted scene", gemm_path, _nets(env, env_id))


# ------------------------------------------------------------------ B. softmax edges
@pytest.mark.parametrize("variant", ["bias+90", "bias-90", "sharp"])
@pytest.mark.parametrize("env_id", ["DoubleIntegrator", "LinearDrone"])
def test_softmax_edges(env_id, variant, gemm_path):
    """Gate bias +-90 (finite, shift-invariant), gate kernel x 50 (near one-hot); the ladder scene has two sender agents
    with identical states (tied logits) in every receiver of degree >= 3."""
    N, area, seed = F.LADDER_SCENE
    env = product_env(env_id, N, area, 0)
    arrays = _synthetic(env_id, N, 1, F.ladder_codes(N, _R(env_id)), seed)
    pre = _net(env, "actor", 1, env_id=env_id)
    nets = [("infer", _variant(pre, variant)), ("forward_l", _variant(pre, variant)),
            ("forward_l", _variant(_net(env, "actor", 2, seed=5), variant))]
    _check(env_id, env, arrays, 0, [0], variant, gemm_path, nets)


# ------------------------------------------------------------------ C. rollout records
def _check_rollout(env_id, env, eng, nets, area, n_obs, what, sample=None):
    """Every recorded action of the sampled environments against 2 pi + u_ref with pi the float64 output of its own
    network (and, with several networks, farther than the bar from every other network's).  u_ref is the float64
    oracle's, but for DubinsCar, whose fp32 u_ref rounding (acos near +-1) exceeds the bar's 3e-6 |u_ref| allowance:
    there it is the library's own (env.u_ref on the rebuilt graph; tests/test_gpu_gnn.py holds it to the oracle's)."""
    c_bar = F.C_BAR_TC if eng.use_tc else F.C_BAR
    T, E = eng.actions.shape[:2]
    N = env.num_agents
    oenv = oracle_env(env_id, N, area, n_obs, dtype=torch.float64)
    table = eng.net_table if len(nets) > 1 else [0] * E
    envs = sorted({0, E // 2, E - 1} | {idx[0] for idx in getattr(eng, "net_envs", [])}) if sample is None else sample
    p64 = [F.params64(n) for n in nets]
    worst, cross = 0.0, float("inf")
    for e in envs:
        obs = eng._obstacle_obj.select([e]) if n_obs > 0 else None
        for t in range(T):
            graph = env.get_graph(eng.agent[t, e][None].contiguous(), eng.goal[e][None].contiguous(), obs,
                                  edge_cap=N * (N + env.n_hits))
            torch.cuda.synchronize()
            graph.check_overflow()
            assert torch.equal(graph.hits, eng.hits[t, e][None]), (e, t)
            og = F.graph_of(oenv, graph)
            u = env.u_ref(graph)[0].cpu().double() if env_id == "DubinsCar" else F.u_ref(oenv, og)
            got = eng.actions[t, e].cpu()
            own = F.forward(p64[table[e]], og, "actor")
            d = F.unit(p64[table[e]], og, "actor", own)
            worst = max(worst, F.action_excess(got, 2 * own + u, u, d, c_bar))
            for k, p in enumerate(p64):
                if k != table[e]:
                    cross = min(cross, F.action_excess(got, 2 * F.forward(p, og, "actor") + u, u, d, c_bar))
    _note(what + " (/bar)", worst, f"{env_id} N={N} E={E} T={T}")
    assert worst <= 1, (what, worst)
    if len(nets) > 1:
        assert cross > 1, (what, cross)


def _engine(env, E, T, n_obs, nets, seed, **kw):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    g0 = env.reset(seed, n_envs=E)
    eng = RolloutEngine(env, E, T=T, n_obs=n_obs, **kw)
    eng.set_params(nets if len(nets) > 1 else nets[0])
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    torch.cuda.synchronize()
    return eng


STEP_CASES = [("DoubleIntegrator", 512, 4, 32.0, 8, 1), ("SingleIntegrator", 8, 16, 4.0, 0, 1),
              ("DubinsCar", 256, 2, 22.63, 16, 1), ("LinearDrone", 1024, 2, 10.08, 4, 1),
              ("DoubleIntegrator", 200, 2, 6.0, 8, 2), ("DoubleIntegrator", 64, 2, 4.0, 8, 3)]


@pytest.mark.parametrize("env_id,N,E,area,n_obs,L", STEP_CASES)
def test_step_path_records(env_id, N, E, area, n_obs, L, gemm_path):
    if L > 1 and gemm_path != "tc":
        pytest.skip("deeper actors run on the tensor-core path only")
    env = product_env(env_id, N, area, n_obs)
    net = _net(env, "actor", 1, env_id=env_id) if L == 1 else _net(env, "actor", L, seed=7)
    eng = _engine(env, E, 2, n_obs, [net], 41, persistent=False)
    assert not eng.persistent and eng.n_layers == L
    _check_rollout(env_id, env, eng, [net], area, n_obs, f"step path L={L} {gemm_path}")


@pytest.mark.parametrize("env_id,N,E,area,n_obs", [("DoubleIntegrator", 512, 16, 32.0, 8),
                                                   ("DoubleIntegrator", 130, 3, 4.0, 3),
                                                   ("SingleIntegrator", 8, 16, 4.0, 0),
                                                   ("DubinsCar", 256, 4, 22.63, 16)])
def test_persistent_records(env_id, N, E, area, n_obs):
    env = product_env(env_id, N, area, n_obs)
    net = _net(env, "actor", 1, env_id=env_id)
    eng = _engine(env, E, 2, n_obs, [net], 43, persistent=True)
    assert eng.persistent and eng.launches_per_run == 1
    _check_rollout(env_id, env, eng, [net], area, n_obs, "persistent")


@pytest.mark.parametrize("N,area,layout", [(512, 32.0, "block"), (130, 4.0, "interleaved")])
def test_multi_network_records(N, area, layout):
    """K = 3 networks in one persistent launch: each environment's actions meet its own network's float64 actions, and
    miss the other two's (a network-table or stride mix-up fails)."""
    env_id, E, n_obs = "DoubleIntegrator", 6, 8
    env = product_env(env_id, N, area, n_obs)
    nets = [_net(env, "actor", 1, seed=s) for s in (1, 2)] + [_net(env, "actor", 1, env_id=env_id)]
    table = None if layout == "block" else [g % 3 for g in range(E)]
    eng = _engine(env, E, 2, n_obs, nets, 47, persistent=True, n_nets=3, net_of_env=table)
    assert eng.persistent and eng.launches_per_run == 1
    _check_rollout(env_id, env, eng, nets, area, n_obs, "multi-network", sample=list(range(E)))


# ------------------------------------------------------------------ D. every GEMM of the unfolded forward
def _saved_activations(ws, cap, A):
    """The activations gcbf_gnn_forward_l (one layer) leaves in its workspace for the backward pass, in the order and
    32-byte slots of make_ws (csrc/gnn.cuh)."""
    sizes = {"feat": cap * 8, "x1": cap * 256, "x2": cap * 256, "msg": cap * 128, "g1": cap * 128, "g2": cap * 128,
             "att": cap, "ag": A * 128, "v1": A * 256, "v2": A * 256, "v3": A * 128, "h1": A * 256, "h2": A * 256}
    out, off = {}, 0
    for name, n in sizes.items():
        out[name] = ws[off:off + n]
        off += (n + 7) & ~7
    return out


def _gemms(p, kind):
    """(layer, input, output, edge rows?, W, b, relu) of every GEMM of the one-layer forward; update/Dense_0 takes the
    aggregate only, its agent one-hot row folded into the bias."""
    g = "params/GNN_0/GNNLayer_0/"
    head = "CBFHead" if kind == "cbf" else "PolicyHead"
    u0 = p[g + "update/Dense_0/kernel"]
    return [("msg/Dense_1", "x1", "x2", True, p[g + "msg/Dense_1/kernel"], p[g + "msg/Dense_1/bias"], False),
            ("Dense_0", "x2", "msg", True, p[g + "Dense_0/kernel"], p[g + "Dense_0/bias"], False),
            ("attn/Dense_0", "msg", "g1", True, p[g + "attn/Dense_0/kernel"], p[g + "attn/Dense_0/bias"], True),
            ("attn/Dense_1", "g1", "g2", True, p[g + "attn/Dense_1/kernel"], p[g + "attn/Dense_1/bias"], False),
            ("update/Dense_0", "ag", "v1", False, u0[3:], p[g + "update/Dense_0/bias"] + u0[2], True),
            ("update/Dense_1", "v1", "v2", False, p[g + "update/Dense_1/kernel"], p[g + "update/Dense_1/bias"], False),
            ("Dense_2", "v2", "v3", False, p[g + "Dense_2/kernel"], p[g + "Dense_2/bias"], False),
            (head + "/Dense_0", "v3", "h1", False, p[f"params/{head}/Dense_0/kernel"],
             p[f"params/{head}/Dense_0/bias"], True),
            (head + "/Dense_1", "h1", "h2", False, p[f"params/{head}/Dense_1/kernel"],
             p[f"params/{head}/Dense_1/bias"], False)]


@pytest.mark.parametrize("case", ["ladder", "one edge", "hub"])
@pytest.mark.parametrize("env_id", ENVS)
def test_every_gemm_of_the_unfolded_forward(env_id, case, gemm_path):
    """Each GEMM output of gcbf_gnn_forward_l against float64 of its own input, in units of 2^-24 (|x| |W| + |b|):
    <= GEMM_BAR on both paths.  A GEMM fed a lost or wrong lo plane (weights at tf32) exceeds it
    (tests/test_gnn_f64_cpu.py), where the network-level bar of the tensor-core path does not tell it from rounding."""
    from gcbfplus_b200 import _lib
    N = {"ladder": 48, "one edge": 64, "hub": 320}[case]
    env = product_env(env_id, N, 2.0, 0)
    degrees = {"ladder": F.LADDER, "one edge": [1] + [0] * (N - 1), "hub": (5,) * 25 + (N + _R(env_id),)}[case]
    arrays = _synthetic(env_id, N, 1, F.ladder_codes(N, _R(env_id), degrees=degrees))
    A, cap, n_edges = N, arrays[5].numel(), int(arrays[7][0])
    for kind in ("actor", "cbf"):
        net = _net(env, kind, 1, env_id=env_id)
        d = env.desc(1, 0, edge_cap=cap)
        out = torch.empty(1, N, net.out_dim, device="cuda")
        ws = torch.zeros(int(env.lib.gcbf_gnn_workspace_floats_l(C.byref(d), net.out_dim, 1)), device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        _lib.check(env.lib.gcbf_gnn_forward_l(
            C.byref(d), _lib.NET_CBF if kind == "cbf" else _lib.NET_ACTOR, net.out_dim, 1, _lib.ptr(net.flat),
            _lib.ptr(net.prepared(st)), *[_lib.ptr(a) for a in arrays], 0, _lib.ptr(out), _lib.ptr(ws), ws.numel(),
            st), "gcbf_gnn_forward_l")
        torch.cuda.synchronize()
        act = _saved_activations(ws.cpu().double(), cap, A)
        worst = []
        for name, xi, yo, edge_rows, w, b, relu in _gemms(F.params64(net), kind):
            M = n_edges if edge_rows else A
            x = act[xi][:M * w.shape[0]].reshape(M, w.shape[0])
            y = act[yo][:M * w.shape[1]].reshape(M, w.shape[1])
            r = F.gemm_ratio(y, x, w, b, relu)
            worst.append((r, name))
        r, name = max(worst)
        _note(f"GEMM {gemm_path}", r, f"{env_id} {case} {kind} worst {name}")
        assert r <= F.GEMM_BAR, (kind, worst)
