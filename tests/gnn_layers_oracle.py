"""Oracle of the multi-layer GNN (TEST INFRASTRUCTURE ONLY): gcbfplus/nn/gnn.py:78-104 with n_layers > 1 restated on
top of oracle/nn.py.  Layer l uses ``params/GNN_0/GNNLayer_<l>/...``; from layer 1 on the node features are the previous
layer's outputs (128 wide), so msg/Dense_0 is [ed + 256, 256] and update/Dense_0 is [256, 256].  Every node row is
computed literally (goal, hit and, in the dense layout, pad nodes too)."""
from __future__ import annotations

import math
from typing import Dict

import numpy as np
import torch

from oracle.envs import Graph
from oracle.nn import _dense, unflatten_params


def layer_specs(edge_dim: int, out_dim: int, kind: str, n_layers: int = 1):
    """(flax path, in, out) in forward order: GNN layers 0 .. n_layers - 1, then the head."""
    specs = []
    for l in range(n_layers):
        g = f"params/GNN_0/GNNLayer_{l}/"
        nd = 3 if l == 0 else 128
        specs += [(g + "msg/Dense_0", edge_dim + 2 * nd, 256), (g + "msg/Dense_1", 256, 256), (g + "Dense_0", 256, 128),
                  (g + "attn/Dense_0", 128, 128), (g + "attn/Dense_1", 128, 128), (g + "Dense_1", 128, 1),
                  (g + "update/Dense_0", nd + 128, 256), (g + "update/Dense_1", 256, 256), (g + "Dense_2", 256, 128)]
    head = "CBFHead" if kind == "cbf" else "PolicyHead"
    last = "Dense_0" if kind == "cbf" else "OutputDense"
    return specs + [(f"params/{head}/Dense_0", 128, 256), (f"params/{head}/Dense_1", 256, 256),
                    (f"params/{last}", 256, out_dim)]


def init_params(edge_dim: int, out_dim: int, kind: str, seed: int, n_layers: int = 1) -> dict:
    """xavier_uniform kernels, zero biases; the NumPy PCG64 stream of NetParams.init_xavier (same draws, same order)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    flat = {}
    for path, fi, fo in layer_specs(edge_dim, out_dim, kind, n_layers):
        lim = math.sqrt(6.0 / (fi + fo))
        flat[path + "/kernel"] = rng.uniform(-lim, lim, size=(fi, fo)).astype(np.float32)
        flat[path + "/bias"] = np.zeros((fo,), dtype=np.float32)
    return unflatten_params(flat)


def n_layers_of(p: Dict[str, torch.Tensor]) -> int:
    n = 0
    while f"params/GNN_0/GNNLayer_{n}/Dense_0/bias" in p:
        n += 1
    return n


def gnn_layer(p: Dict[str, torch.Tensor], l: int, nodes, edges, senders, receivers):
    """nn/gnn.py:22-75 for GNN layer l.  Returns new node features [n_nodes, 128]."""
    g = f"params/GNN_0/GNNLayer_{l}/"
    n_nodes = nodes.shape[0]
    feats = torch.cat([edges, nodes[senders], nodes[receivers]], dim=-1)
    x = torch.relu(_dense(p, g + "msg/Dense_0", feats))
    x = _dense(p, g + "msg/Dense_1", x)
    msg = _dense(p, g + "Dense_0", x)
    gf = torch.relu(_dense(p, g + "attn/Dense_0", msg))
    gf = _dense(p, g + "attn/Dense_1", gf)
    gate = _dense(p, g + "Dense_1", gf).squeeze(-1)
    seg_max = torch.full((n_nodes,), -float("inf"), dtype=gate.dtype)
    seg_max = seg_max.scatter_reduce(0, receivers, gate.detach(), reduce="amax", include_self=True)
    ex = torch.exp(gate - seg_max[receivers])
    denom = torch.zeros(n_nodes, dtype=gate.dtype).index_add(0, receivers, ex)
    attn = ex / denom[receivers]
    aggr = torch.zeros(n_nodes, msg.shape[1], dtype=msg.dtype).index_add(0, receivers, attn[:, None] * msg)
    u = torch.cat([nodes, aggr], dim=-1)
    u = torch.relu(_dense(p, g + "update/Dense_0", u))
    u = _dense(p, g + "update/Dense_1", u)
    return _dense(p, g + "Dense_2", u)


def net_forward(p: Dict[str, torch.Tensor], graph: Graph, kind: str) -> torch.Tensor:
    """CBFNet / Deterministic with every GNNLayer_<l> of `p` applied in turn, then the head on the agent rows."""
    x = graph.nodes.to(p["params/GNN_0/GNNLayer_0/Dense_0/bias"].dtype)
    for l in range(n_layers_of(p)):
        x = gnn_layer(p, l, x, graph.edges, graph.senders, graph.receivers)
    x = x[: graph.n_agents]
    head = "CBFHead" if kind == "cbf" else "PolicyHead"
    last = "Dense_0" if kind == "cbf" else "OutputDense"
    x = torch.relu(_dense(p, f"params/{head}/Dense_0", x))
    x = _dense(p, f"params/{head}/Dense_1", x)
    return torch.tanh(_dense(p, f"params/{last}", x))
