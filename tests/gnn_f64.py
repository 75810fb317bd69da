"""Float64 reference of the product's GNN forwards on a device graph (TEST INFRASTRUCTURE ONLY).

`oracle_graph` turns one graph of the product's arrays (agent, goal, hits, row_start, row_deg, edge_recv, edge_src,
counters, clip_all) into an `oracle.envs.Graph` in float64 with exactly the edges the device lists name; the edge
features are the oracle's own (its dense get_graph computes every (receiver, sender) pair, masked or not, and
add_edge_feats gives the clip_all features).  `forward` / `act` are the oracle's networks in float64.

The bar.  `unit` is the size of fp32 rounding for one case: the largest change of the float64 output when every weight,
bias and edge feature is perturbed by a relative +-2^-24 (uniform, 4 seeds, max).  A CUDA output passes when
|got - f64| <= C_BAR * unit per output tensor.  On the CPU (tests/test_gnn_f64_cpu.py) the float32 oracle sits at
1-18 units, rounding the weights of any one layer to tf32 (a lost lo plane, or a wrong hi / lo split, in one GEMM)
moves the output by > 32 units but for three layers of the pretrained SingleIntegrator CBF (4-18 units), and dropping
one edge moves the receiver's output by a median of thousands of units (a sender with a negligible attention weight
excepted).  The tensor-core path is held to C_BAR_TC per output and to GEMM_BAR per GEMM (below).
"""
from __future__ import annotations

from contextlib import contextmanager
from dataclasses import replace

import numpy as np
import torch

import gnn_layers_oracle
import oracle.nn
from gnn_layers_oracle import n_layers_of
from gnn_layers_oracle import net_forward as net_forward_l
from oracle.envs import Graph, OracleEnv
from oracle.nn import net_forward as net_forward_1
from oracle.nn import to_torch

C_BAR = 32
#: The wgmma tensor-core path: its fp32 accumulation truncates (tc_dense reproduces gcbf_gemm_tc's error), so each of
#: its GEMM outputs carries up to 25 units of 2^-24 (|x| |W| + |b|) where the SIMT GEMM carries <= 10 (measured on an
#: NVIDIA H100 80GB HBM3 at 700 W, with exact accumulation of the same split operands at <= 1).  That puts its network
#: outputs at up to 72 units (gcbf_gnn_infer) and 260 (gcbf_gnn_forward_l) of the fp32 unit above.  Its network-level bar C_BAR_TC catches structural errors (a lost or
#: extra row, a misread tile); a GEMM at the wrong precision is caught per GEMM instead, in the GEMM's own unit, by
#: GEMM_BAR.
C_BAR_TC = 10 * C_BAR
GEMM_BAR = 48
U = 2.0 ** -24
F64 = torch.float64


def params64(net) -> dict:
    """Float64 flat dict of a NetParams (device) or a nested parameter tree."""
    tree = net.to_tree() if hasattr(net, "to_tree") else net
    return to_torch(tree, F64)


def _np(x, dtype=None):
    a = x.detach().cpu().numpy() if torch.is_tensor(x) else np.asarray(x)
    return a if dtype is None else a.astype(dtype)


def oracle_graph(oenv: OracleEnv, agent, goal, hits, row_start, row_deg, edge_recv, edge_src, counters,
                 clip_all: int = 0, g: int = 0) -> Graph:
    """Graph g of a device batch (agent / goal [G, N, sd], hits [G, N, R, pd], int32 lists over the whole batch) as a
    float64 oracle Graph.  Sender codes: >= 0 global agent id, -1 the receiver's goal, -2 - k the receiver's hit k.
    Only rows the receivers' [row_start, row_start + row_deg) ranges name are read; they must lie below counters[0]."""
    N, R, sd, pd = oenv.num_agents, oenv.n_hits, oenv.state_dim, oenv.pos_dim
    a64 = torch.from_numpy(_np(agent, np.float64)[g])
    g64 = torch.from_numpy(_np(goal, np.float64)[g])
    lidar = torch.zeros(N, R, sd, dtype=F64)
    lidar[..., :pd] = torch.from_numpy(_np(hits, np.float64)[g])
    dense = oenv.get_graph(a64, g64, None, lidar=lidar)
    n_goal_rows = dense.edges.shape[0] - N * N - N * R     # N * N (eye-masked block), or N (DubinsCar: one row each)
    rs = _np(row_start, np.int64)[g * N:(g + 1) * N]
    rd = _np(row_deg, np.int64)[g * N:(g + 1) * N]
    recv_all, src_all = _np(edge_recv, np.int64), _np(edge_src, np.int64)
    n_edges = int(_np(counters)[0])
    assert (rs >= 0).all() and (rd >= 0).all() and (rs + rd <= n_edges).all(), "rows beyond the edge counter"
    recv = np.repeat(np.arange(N), rd)
    rows = np.concatenate([np.arange(s, s + d) for s, d in zip(rs, rd)]) if rd.sum() else np.zeros(0, np.int64)
    assert (recv_all[rows] == recv + g * N).all(), "edge_recv disagrees with the row ranges"
    code = src_all[rows]
    is_agent, is_goal = code >= 0, code == -1
    j = code - g * N
    k = -2 - code
    assert (j[is_agent] >= 0).all() and (j[is_agent] < N).all(), "sender agent outside the receiver's graph"
    assert (k[~is_agent & ~is_goal] < R).all(), "hit code beyond n_hits"
    goal_row = N * N + (recv * N + recv if n_goal_rows == N * N else recv)
    dense_row = np.where(is_agent, recv * N + j, np.where(is_goal, goal_row, N * N + n_goal_rows + recv * R + k))
    sender = np.where(is_agent, j, np.where(is_goal, N + recv, 2 * N + recv * R + k))
    out = replace(dense, edges=dense.edges[torch.from_numpy(dense_row)], receivers=torch.from_numpy(recv),
                  senders=torch.from_numpy(sender))
    if clip_all:
        out = oenv.add_edge_feats(out, dense.states[:-1])
    return out


def graph_of(oenv, graph, g: int = 0, clip_all=None) -> Graph:
    """oracle_graph of graph g of a product SwarmGraph."""
    return oracle_graph(oenv, graph.agent, graph.goal, graph.hits, graph.row_start, graph.row_deg, graph.edge_recv,
                        graph.edge_src, graph.counters, int(graph.clip_all if clip_all is None else clip_all), g)


def forward(p: dict, graph: Graph, kind: str) -> torch.Tensor:
    """The oracle's CBF / actor network in the dtype of `p` (oracle.nn at one GNN layer, gnn_layers_oracle deeper)."""
    with torch.no_grad():
        return (net_forward_1 if n_layers_of(p) == 1 else net_forward_l)(p, graph, kind)


def act(oenv: OracleEnv, p: dict, graph: Graph) -> torch.Tensor:
    """oracle.algo.act in float64: 2 pi + u_ref, unclipped (what the rollout records)."""
    return 2 * forward(p, graph, "actor") + u_ref(oenv, graph)


def u_ref(oenv: OracleEnv, graph: Graph) -> torch.Tensor:
    return oenv.u_ref(graph.agent, graph.goal)


def perturbed(p: dict, seed: int, rel: float = U) -> dict:
    gen = torch.Generator().manual_seed(seed)
    return {k: v * (1 + rel * (2 * torch.rand(v.shape, generator=gen, dtype=v.dtype) - 1)) for k, v in p.items()}


@contextmanager
def dense_as(fn):
    """Run the oracle networks with `fn(p, path, x)` in place of every dense layer."""
    saved = oracle.nn._dense, gnn_layers_oracle._dense
    oracle.nn._dense = gnn_layers_oracle._dense = fn
    try:
        yield
    finally:
        oracle.nn._dense, gnn_layers_oracle._dense = saved


def unit(p: dict, graph: Graph, kind: str, ref=None, seeds: int = 4) -> float:
    """The fp32 rounding unit of one case: max |f(p', graph') - f(p, graph)| over `seeds` draws of p' (every weight and
    bias) and graph' (every edge feature) perturbed by a relative +-2^-24."""
    ref = forward(p, graph, kind) if ref is None else ref
    d = 0.0
    for s in range(seeds):
        gen = torch.Generator().manual_seed(1000 + s)
        e = graph.edges * (1 + U * (2 * torch.rand(graph.edges.shape, generator=gen, dtype=graph.edges.dtype) - 1))
        d = max(d, float((forward(perturbed(p, s), replace(graph, edges=e), kind) - ref).abs().max()))
    return d


def gemm_ratio(y, x, w, b, relu=False) -> float:
    """max |y - epi(x W + b)| of one dense layer in its own unit, 2^-24 (|x| |W| + |b|) per element (float64 from the
    layer's own input x)."""
    pre = x @ w + b
    ref = torch.relu(pre) if relu else pre
    return float(((y - ref).abs() / (U * (x.abs() @ w.abs() + b.abs()) + 1e-300)).max())


def tc_dense(p, path, x):
    """A dense layer as the wgmma 3xTF32 GEMM computes it: operands split into rn-tf32 hi + lo (lo x lo dropped); per
    k8 step the three MMAs (lo hi, hi lo, hi hi) each add 8 exact products to the fp32 accumulator with every term
    truncated to a 26-bit window below the largest one and the sum rounded toward zero to fp32.  On an H100 this
    model reproduces gcbf_gemm_tc's error on a 1024 x 256 x 256 product (max 20.9 / 21.7, mean +0.16 / +0.17,
    rms 4.19 / 4.18 units of 2^-24 |A| |B|), where exact accumulation of the same operands gives rms 0.16."""
    w, b = p[path + "/kernel"], p[path + "/bias"]
    xh = _rn_tf32(x)
    xl = _rn_tf32(x - xh)
    wh = _rn_tf32(w)
    wl = _rn_tf32(w - wh)
    acc = torch.zeros(x.shape[0], w.shape[1], dtype=F64)
    K = w.shape[0]
    for k0 in range(0, K, 8):
        k1 = min(k0 + 8, K)
        for a, m in ((xl, wh), (xh, wl), (xh, wh)):
            terms = torch.cat([a[:, k0:k1].T[:, :, None] * m[k0:k1, None, :], acc[None]], 0)
            q = torch.pow(2.0, torch.frexp(terms.abs().amax(0))[1].double() - 26)
            s = torch.trunc(terms / q).sum(0) * q
            q = torch.pow(2.0, torch.frexp(s.abs())[1].double() - 24)
            acc = torch.trunc(s / q) * q
    return (acc + b).float().double()


def _rn_tf32(t):
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).double()


def ratio(got, want, delta: float) -> float:
    """max |got - want| in units of delta (inf for a non-finite output)."""
    got = torch.as_tensor(_np(got, np.float64))
    if not torch.isfinite(got).all():
        return float("inf")
    return float((got - want).abs().max()) / delta


def action_excess(got, want, u, delta_pi: float, c_bar: float = C_BAR) -> float:
    """max |got - want| / (2 c_bar delta_pi + 2e-6 + 3e-6 |u_ref|): <= 1 passes the action bar."""
    got = torch.as_tensor(_np(got, np.float64))
    if not torch.isfinite(got).all():
        return float("inf")
    return float(((got - want).abs() / (2 * c_bar * delta_pi + 2e-6 + 3e-6 * u.abs())).max())


# --------------------------------------------------------------------------- device-format edge lists
def write_rows(codes, N: int, order=None, cap=None):
    """Device edge lists from per-receiver sender codes.  codes[a] (a = global receiver, G * N of them) lists the
    receiver's senders as j >= 0 (agent j of its own graph), -1 (its goal) or -2 - k (its hit k); the rows of the
    receivers are written one receiver after another in `order` (default: ascending).  Rows [n_edges, cap) are slack:
    valid but wrong rows (a same-graph agent sending to an agent), which a kernel reading past the edge counter turns
    into wrong numbers.  Returns int32 row_start, row_deg, edge_recv, edge_src [cap], counters [4]."""
    A = len(codes)
    order = range(A) if order is None else order
    row_start, row_deg = np.zeros(A, np.int32), np.zeros(A, np.int32)
    recv, src = [], []
    for a in order:
        row_start[a], row_deg[a] = len(recv), len(codes[a])
        base = (a // N) * N
        recv += [a] * len(codes[a])
        src += [c + base if c >= 0 else c for c in codes[a]]
    n = len(recv)
    cap = n if cap is None else cap
    assert cap >= n
    for e in range(n, cap):
        a = e % A
        recv.append(a)
        src.append((a // N) * N + (a % N + 1 + e % 7) % N)
    return (row_start, row_deg, np.asarray(recv, np.int32), np.asarray(src, np.int32),
            np.array([n, 0, 0, 0], np.int32))


def canonical_codes(og: Graph):
    """Per-receiver sender codes of an oracle sparse graph in the canonical row order [goal | agents ascending |
    hits ascending]."""
    N, R = og.n_agents, og.n_hits
    codes = [[] for _ in range(N)]
    for r, s in sorted(zip(og.receivers.tolist(), og.senders.tolist())):
        codes[r].append(s if s < N else (-1 if s < 2 * N else -2 - (s - 2 * N - r * R)))
    return [sorted(c, key=lambda c: (c != -1, c < -1, c if c >= 0 else -c)) for c in codes]


LADDER = (1, 2, 3, 4, 5, 6, 8, 31, 32, 33, 64)
LADDER_SCENE = (48, 2.0, 3)      # N, area, seed of the degree-ladder graphs


def softmax_variants(p: dict) -> dict:
    """The softmax edges of GNN layer 0: gate bias shifted to +90 / -90 (shift-invariant in exact arithmetic, NaN
    without the max subtraction) and the gate kernel scaled by 50 (nearly one-hot attention)."""
    g = "params/GNN_0/GNNLayer_0/Dense_1/"
    out = {}
    for name, b in (("bias+90", 90.0), ("bias-90", -90.0)):
        out[name] = dict(p)
        out[name][g + "bias"] = torch.full_like(p[g + "bias"], b)
    out["sharp"] = dict(p)
    out["sharp"][g + "kernel"] = p[g + "kernel"] * 50
    return out


def ladder_codes(N: int, R: int, G: int = 1, degrees=LADDER, seed: int = 0):
    """Synthetic sender codes: in every graph agent i < len(degrees) receives degrees[i] rows (goal, then agents, then
    hits; none for degree 0), the others 1 to 6 rows; needs N + R >= max(degrees)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    codes = []
    for _ in range(G):
        for i in range(N):
            d = degrees[i] if i < len(degrees) else int(rng.integers(1, 7))
            if d == 0:
                codes.append([])
                continue
            # agents N - 2 and N - 1 have identical states (synthetic_scene): every receiver of degree >= 3 lists both
            first = [N - 2, N - 1] if d >= 3 and i < N - 2 else []
            others = first + [j for j in rng.permutation(N).tolist() if j != i and j not in first]
            n_ag = min(d - 1, N - 1, max(d - 1 - R, (d - 1 + 1) // 2))
            c = [-1] + sorted(others[:n_ag]) + sorted(-2 - k for k in rng.permutation(R)[:d - 1 - n_ag].tolist())[::-1]
            assert len(c) == d
            codes.append(c)
    return codes


def synthetic_scene(env_id: str, N: int, G: int, area: float, seed: int):
    """States for synthetic edge lists: random agents / goals and hit points 0.05-0.4 from their agent (hits are an
    input of the forward, so every hit code names a plausible nearby obstacle point)."""
    from helpers import random_scene
    agent, goal, _ = random_scene(env_id, N, G, area, 0, seed)
    pd = 3 if env_id == "LinearDrone" else 2
    R = 16 if env_id in ("DubinsCar", "LinearDrone") else 32     # the oracle's (and the product's) n_hits
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    v = rng.normal(size=(G, N, R, pd))
    v *= (rng.uniform(0.05, 0.4, size=(G, N, R, 1)) / np.linalg.norm(v, axis=-1, keepdims=True))
    hits = (agent[:, :, None, :pd] + v).astype(np.float32)
    agent[:, N - 1], goal[:, N - 1], hits[:, N - 1] = agent[:, N - 2], goal[:, N - 2], hits[:, N - 2]   # tied logits
    return agent, goal, hits
