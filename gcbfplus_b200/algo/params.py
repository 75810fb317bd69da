"""Network parameters: flat fp32 device buffers <-> the reference's nested flax dict.

Layout of one network (CBF or actor) = the 12 Dense layers in forward order
(gcbfplus/nn/gnn.py:44-104, algo/module/cbf.py:12-53, algo/module/policy.py:63-128;
names per SURVEY A.3), kernel [in, out] row-major then bias, each 16-byte aligned;
offsets come from libgcbf_b200 (gcbf_param_offsets_l) so C and Python cannot drift.
With n_layers GNN layers (gnn.py:78-104) the 9 Dense layers of GNNLayer_0 .. GNNLayer_<n-1> come first, then the
head.
Checkpoints keep the reference format: pickle of {'params': nested dict} with NumPy leaves
(gcbfplus/algo/gcbf.py:344-357); the reference's own pickles (jax.Array leaves) load
through a stub unpickler, no JAX needed.
"""
from __future__ import annotations

import math
import pickle
from typing import Dict, List, Tuple

import numpy as np
import torch

from .. import _lib


def layer_specs(edge_dim: int, out_dim: int, kind: str, n_layers: int = 1) -> List[Tuple[str, int, int]]:
    """(flax path, in, out) in forward order.  Layer 0 reads the 3-wide one-hot node types; every later layer reads the
    previous layer's 128-wide output, so its msg/Dense_0 is [ed + 256, 256] and its update/Dense_0 [256, 256]."""
    specs = []
    for l in range(n_layers):
        g = f"params/GNN_0/GNNLayer_{l}/"
        nd = 3 if l == 0 else 128
        specs += [
            (g + "msg/Dense_0", edge_dim + 2 * nd, 256), (g + "msg/Dense_1", 256, 256), (g + "Dense_0", 256, 128),
            (g + "attn/Dense_0", 128, 128), (g + "attn/Dense_1", 128, 128), (g + "Dense_1", 128, 1),
            (g + "update/Dense_0", nd + 128, 256), (g + "update/Dense_1", 256, 256), (g + "Dense_2", 256, 128),
        ]
    head = "CBFHead" if kind == "cbf" else "PolicyHead"
    last = "Dense_0" if kind == "cbf" else "OutputDense"
    return specs + [
        (f"params/{head}/Dense_0", 128, 256), (f"params/{head}/Dense_1", 256, 256),
        (f"params/{last}", 256, out_dim),
    ]


def flatten_tree(tree: dict, prefix: str = "") -> Dict[str, np.ndarray]:
    out = {}
    for k, v in tree.items():
        if isinstance(v, dict):
            out.update(flatten_tree(v, prefix + k + "/"))
        else:
            out[prefix + k] = np.asarray(v)
    return out


def unflatten_tree(flat: Dict[str, np.ndarray]) -> dict:
    tree: dict = {}
    for k, v in flat.items():
        parts = k.split("/")
        d = tree
        for p in parts[:-1]:
            d = d.setdefault(p, {})
        d[parts[-1]] = v
    return tree


class _RefUnpickler(pickle.Unpickler):
    """Reads reference checkpoints whose leaves are pickled jax.Array objects."""

    def find_class(self, module, name):
        if module.startswith("jax") and name == "_reconstruct_array":
            def rec(fun, args, arr_state, aval_state):
                arr = fun(*args)
                arr.__setstate__(arr_state)
                return arr
            return rec
        if module.startswith("numpy.core"):
            module = module.replace("numpy.core", "numpy._core")
        return super().find_class(module, name)


def load_pickle(path: str) -> dict:
    with open(path, "rb") as f:
        return _RefUnpickler(f).load()


class NetParams:
    """One network's parameters as a flat fp32 device buffer."""

    def __init__(self, edge_dim: int, out_dim: int, kind: str, device="cuda", n_layers: int = 1):
        assert kind in ("cbf", "actor")
        self.edge_dim, self.out_dim, self.kind, self.n_layers = edge_dim, out_dim, kind, n_layers
        self.specs = layer_specs(edge_dim, out_dim, kind, n_layers)
        self.offsets = _lib.param_offsets(edge_dim, out_dim, n_layers)
        self.count = _lib.param_count(edge_dim, out_dim, n_layers)
        self.flat = torch.zeros(self.count, dtype=torch.float32, device=device)
        self._flat_t = None   # tf32 planes of the GEMM weights for the tensor-core path (gcbf_prepare_params_l)

    def prepared(self, stream: int = None):
        """Transposed GEMM weights (K-major B operands of the wgmma path), recomputed from `flat`.
        Returns None when the tensor-core path is disabled (GCBF_TENSOR_CORES=0)."""
        if not _lib.USE_TC:
            return None
        lib = _lib.load()
        if self._flat_t is None:
            n = lib.gcbf_params_t_count_l(self.edge_dim, self.out_dim, self.n_layers)
            self._flat_t = torch.empty(int(n), dtype=torch.float32, device=self.flat.device)
        if stream is None:
            stream = torch.cuda.current_stream(self.flat.device).cuda_stream
        _lib.check(lib.gcbf_prepare_params_l(self.edge_dim, self.out_dim, self.n_layers, _lib.ptr(self.flat),
                                             _lib.ptr(self._flat_t), stream), "gcbf_prepare_params_l")
        return self._flat_t

    # ---- init (nn/utils.py:21 xavier_uniform kernels, zero biases) ----
    def init_xavier(self, seed: int) -> "NetParams":
        rng = np.random.Generator(np.random.PCG64(seed))
        host = np.zeros(self.count, dtype=np.float32)
        for i, (_, fi, fo) in enumerate(self.specs):
            lim = math.sqrt(6.0 / (fi + fo))
            w = rng.uniform(-lim, lim, size=(fi, fo)).astype(np.float32)
            host[self.offsets[2 * i]: self.offsets[2 * i] + fi * fo] = w.reshape(-1)
        self.flat.copy_(torch.from_numpy(host))
        return self

    # ---- nested dict <-> flat ----
    def from_tree(self, tree: dict) -> "NetParams":
        flat = flatten_tree(tree)
        known = {path for path, _, _ in self.specs}
        extra = sorted({k.rsplit("/", 1)[0] for k in flat if "/GNNLayer_" in k} - known)
        if extra:   # a deeper network's checkpoint: loading its first layers only would silently drop the rest
            raise ValueError(f"checkpoint has GNN layers this {self.n_layers}-layer network lacks: {extra[0]} ...")
        host = np.zeros(self.count, dtype=np.float32)
        for i, (path, fi, fo) in enumerate(self.specs):
            w = np.asarray(flat[path + "/kernel"], dtype=np.float32)
            b = np.asarray(flat[path + "/bias"], dtype=np.float32)
            if w.shape != (fi, fo) or b.shape != (fo,):
                raise ValueError(f"{path}: expected kernel {(fi, fo)}, got {w.shape}")
            host[self.offsets[2 * i]: self.offsets[2 * i] + fi * fo] = w.reshape(-1)
            host[self.offsets[2 * i + 1]: self.offsets[2 * i + 1] + fo] = b
        self.flat.copy_(torch.from_numpy(host))
        return self

    def to_tree(self) -> dict:
        host = self.flat.detach().cpu().numpy()
        flat = {}
        for i, (path, fi, fo) in enumerate(self.specs):
            flat[path + "/kernel"] = host[self.offsets[2 * i]: self.offsets[2 * i] + fi * fo].reshape(fi, fo).copy()
            flat[path + "/bias"] = host[self.offsets[2 * i + 1]: self.offsets[2 * i + 1] + fo].copy()
        return unflatten_tree(flat)

    def n_real(self) -> int:
        return sum(fi * fo + fo for _, fi, fo in self.specs)

    def clone(self) -> "NetParams":
        out = NetParams(self.edge_dim, self.out_dim, self.kind, device=self.flat.device, n_layers=self.n_layers)
        out.flat.copy_(self.flat)
        return out

    def save(self, path: str) -> None:
        with open(path, "wb") as f:
            pickle.dump(self.to_tree(), f)

    def load(self, path: str) -> "NetParams":
        return self.from_tree(load_pickle(path))
