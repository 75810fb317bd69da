"""GCBF+ update -- host orchestration of gcbfplus/algo/gcbf_plus.py:198-297,354-447
(update, sample_batch, update_nets, update_inner) on top of libgcbf_b200's train-step kernels.

Per minibatch: gcbf_mask_counts -> [all-reduce counts] -> gcbf_train_step -> [ONE all-reduce of
(grad_cbf | grad_actor | stats)] -> gcbf_grad_sqnorm + gcbf_clip_adamw per network.  No host
synchronisation inside the minibatch loop; the info dict of the LAST minibatch is read back
once per epoch loop (the reference returns the last minibatch's info, gcbf_plus.py:445-446).
"""
from __future__ import annotations

import ctypes as C
import os
from typing import Dict, Optional

import numpy as np
import torch

from .. import _lib
from ..trainer.buffer import MaskedReplayBuffer
from ..trainer.data import Rollout
from ..utils.graph import SwarmGraph


class TrainState:
    """Optimizer state + packed gradient buffer for both networks (flax TrainState analogue)."""

    def __init__(self, algo):
        dev = algo._env.device
        self.n_cbf = algo.cbf_params.count
        self.n_act = algo.actor_net_params.count
        f32 = torch.float32
        # one contiguous buffer so that a sharded run needs ONE all-reduce per optimizer step
        self.packed = torch.zeros(self.n_cbf + self.n_act + 16, dtype=f32, device=dev)
        self.grad_cbf = self.packed[: self.n_cbf]
        self.grad_act = self.packed[self.n_cbf: self.n_cbf + self.n_act]
        self.stats = self.packed[self.n_cbf + self.n_act:]
        self.m_cbf = torch.zeros(self.n_cbf, dtype=f32, device=dev)
        self.v_cbf = torch.zeros(self.n_cbf, dtype=f32, device=dev)
        self.m_act = torch.zeros(self.n_act, dtype=f32, device=dev)
        self.v_act = torch.zeros(self.n_act, dtype=f32, device=dev)
        self.step_cbf = torch.zeros(1, dtype=torch.int32, device=dev)
        self.step_act = torch.zeros(1, dtype=torch.int32, device=dev)
        self.norm_cbf = torch.zeros(2 + 512, dtype=f32, device=dev)
        self.norm_act = torch.zeros(2 + 512, dtype=f32, device=dev)
        self.denoms = torch.zeros(4, dtype=f32, device=dev)
        # sticky OR of the edge-capacity overflow flag (counters[1]) of every graph trained on / labelled since the
        # last read_info(): an overflowed build drops rows, which must never train silently
        self.overflow = torch.zeros(1, dtype=torch.int32, device=dev)
        self.ws: Optional[torch.Tensor] = None
        self.ws_key = None


def _dist():
    import torch.distributed as dist
    if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
        return dist
    return None


def train_minibatch(algo, graph: SwarmGraph, safe_mask: torch.Tensor, unsafe_mask: torch.Tensor,
                    u_qp: torch.Tensor, apply: bool = True, denoms_ready: bool = False) -> TrainState:
    """One `update_fn` (gcbf_plus.py:356-441) on the (local shard of the) minibatch `graph`.
    safe/unsafe_mask uint8 [B, N]; u_qp [B, N, nu].  Enqueues only (no host sync).
    denoms_ready: ts.denoms already holds the GLOBAL label counts of this minibatch (update() all-reduces the counts
    of a whole epoch's minibatches in one collective, SURVEY 8e) -> no count kernel, no count all-reduce here."""
    env = algo._env
    lib = env.lib
    if algo._trainer_state is None:
        algo._trainer_state = TrainState(algo)
    ts: TrainState = algo._trainer_state
    B, N = graph.n_graphs, env.num_agents
    d = env.desc(B, 0, edge_cap=graph.edge_recv.numel())
    key = (B, d.edge_cap)
    if ts.ws_key != key:
        n = lib.gcbf_train_workspace_floats(C.byref(d))
        if n <= 0:
            raise RuntimeError("gcbf_train_workspace_floats failed")
        ts.ws = None
        ts.ws = torch.empty(int(n), dtype=torch.float32, device=env.device)
        ts.ws_key = key
    st = env._stream()
    ts.overflow |= graph.counters[1:2]
    safe_mask = safe_mask.reshape(B * N).to(torch.uint8).contiguous()
    unsafe_mask = unsafe_mask.reshape(B * N).to(torch.uint8).contiguous()
    u_qp = u_qp.reshape(B * N, env.action_dim).float().contiguous()
    dist = _dist()
    if not denoms_ready:
        _lib.check(lib.gcbf_mask_counts(_lib.ptr(safe_mask), _lib.ptr(unsafe_mask), B * N, _lib.ptr(ts.denoms), st),
                   "gcbf_mask_counts")
        if dist is not None:
            dist.all_reduce(ts.denoms)                  # global ratio-of-sums denominators (SURVEY 8e)
    hp = (C.c_float * 7)(algo.alpha, algo.eps, algo.loss_action_coef, algo.loss_unsafe_coef, algo.loss_safe_coef,
                         algo.loss_h_dot_coef, 1.0 if _lib.USE_TC else 0.0)
    rc = lib.gcbf_train_step(C.byref(d), hp, _lib.ptr(algo.cbf_params.flat), _lib.ptr(algo.actor_net_params.flat),
                             _lib.ptr(graph.agent), _lib.ptr(graph.goal), _lib.ptr(graph.hits),
                             _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_recv),
                             _lib.ptr(graph.edge_src), _lib.ptr(graph.counters), _lib.ptr(safe_mask),
                             _lib.ptr(unsafe_mask), _lib.ptr(u_qp), _lib.ptr(ts.denoms), _lib.ptr(ts.grad_cbf),
                             _lib.ptr(ts.grad_act), _lib.ptr(ts.stats), _lib.ptr(ts.ws), ts.ws.numel(), st)
    _lib.check(rc, "gcbf_train_step")
    if dist is not None:
        dist.all_reduce(ts.packed)                      # the single gradient all-reduce per optimizer step
    if apply:
        apply_gradients(algo, ts)
    return ts


class MinibatchRunner:
    """One optimizer step of update_inner as ONE CUDA-graph replay (VERDICT r1 #4).

    Captured once per (minibatch size, edge capacity, batch storage): gather of the selected graphs out of the update's
    batch arrays into static buffers -> neighbour lists (gcbf_graph_build, topology only) -> gcbf_train_step ->
    [the ONE NCCL all-reduce of (grad_cbf | grad_actor | stats)] -> grad norm + clip + AdamW for both networks.
    Per minibatch the host then does two tiny device copies (selection indices, global label counts) and one graph
    launch instead of ~170 kernel launches with per-launch tensor-map encoding: the train step stops being bound by
    Python / launch overhead when a rank's share of the minibatch is small (8 GPUs: 32 graphs per rank).
    GCBF_TRAIN_GRAPH=0 keeps the eager path (same kernels, same order -> same bits: the graph build's canonical edge
    layout and the train step's fixed-order reductions make every launch deterministic)."""

    def __init__(self, algo, batch: dict, mb_size: int, edge_cap: int, u_qp: torch.Tensor):
        env = algo._env
        dev = env.device
        self.algo, self.batch, self.u_qp_all = algo, batch, u_qp
        N = env.num_agents
        self.sel = torch.zeros(mb_size, dtype=torch.int64, device=dev)
        self.agent = torch.zeros(mb_size, N, env.state_dim, dtype=torch.float32, device=dev)
        self.goal = torch.zeros_like(self.agent)
        self.hits = torch.zeros(mb_size, N, env.n_hits, env.pos_dim, dtype=torch.float32, device=dev)
        self.safe = torch.zeros(mb_size, N, dtype=batch["safe"].dtype, device=dev)
        self.unsafe = torch.zeros(mb_size, N, dtype=batch["unsafe"].dtype, device=dev)
        self.u_qp = torch.zeros(mb_size, N, env.action_dim, dtype=torch.float32, device=dev)
        i32 = torch.int32
        cap = max(int(edge_cap), 64)
        self.graph = SwarmGraph(env, self.agent, self.goal, None, self.hits,
                                torch.zeros(mb_size * N, dtype=i32, device=dev), torch.zeros(mb_size * N, dtype=i32, device=dev),
                                torch.zeros(cap, dtype=i32, device=dev), torch.zeros(cap, dtype=i32, device=dev),
                                torch.zeros(4, dtype=i32, device=dev))
        self.cuda_graph: Optional[torch.cuda.CUDAGraph] = None

    def _body(self) -> None:
        algo, env, b = self.algo, self.algo._env, self.batch
        torch.index_select(b["agent"], 0, self.sel, out=self.agent)
        torch.index_select(b["goal"], 0, self.sel, out=self.goal)
        torch.index_select(b["hits"], 0, self.sel, out=self.hits)
        torch.index_select(b["safe"], 0, self.sel, out=self.safe)
        torch.index_select(b["unsafe"], 0, self.sel, out=self.unsafe)
        torch.index_select(self.u_qp_all, 0, self.sel, out=self.u_qp)
        env.get_graph(self.agent, self.goal, None, hits=self.hits, out=self.graph)
        train_minibatch(algo, self.graph, self.safe, self.unsafe, self.u_qp, apply=True, denoms_ready=True)

    def run(self, sel: torch.Tensor, denoms: torch.Tensor) -> None:
        ts: TrainState = self.algo._trainer_state
        self.sel.copy_(sel, non_blocking=True)
        ts.denoms.copy_(denoms, non_blocking=True)
        if os.environ.get("GCBF_TRAIN_GRAPH", "1") == "0":
            self._body()
            return
        if self.cuda_graph is None:
            self._body()                                   # warm-up outside capture: function attributes, workspaces,
            torch.cuda.synchronize(self.agent.device)      # NCCL communicator setup
            # (the warm-up was a real optimizer step on this minibatch; the capture below records, it does not run)
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._body()
            self.cuda_graph = g
            return
        self.cuda_graph.replay()


def _minibatch_counts(batch: dict, idx: torch.Tensor, bounds: np.ndarray) -> torch.Tensor:
    """[n_mb, 4] = (n_unsafe, n_safe, n_agents, 0) of every minibatch idx[bounds[i]:bounds[i+1]] of an epoch, on the
    device, without a loop: per-graph counts -> permute -> cumulative sums at the split points."""
    N = batch["safe"].shape[1]
    per = torch.stack([batch["unsafe"].reshape(len(idx), -1).float().sum(1), batch["safe"].reshape(len(idx), -1).float().sum(1)],
                      dim=1)[idx]                                               # [n, 2] in minibatch order
    cs = torch.cat([torch.zeros(1, 2, device=per.device, dtype=torch.float64), per.double().cumsum(0)])
    b = torch.from_numpy(bounds).to(per.device)
    cnt = (cs[b[1:]] - cs[b[:-1]]).float()
    n_ag = ((b[1:] - b[:-1]) * N).float()[:, None]
    return torch.cat([cnt, n_ag, torch.zeros_like(n_ag)], dim=1).contiguous()


def apply_gradients(algo, ts: TrainState) -> None:
    """compute_norm_and_clip + TrainState.apply_gradients for both nets (gcbf_plus.py:435-438)."""
    lib = algo._env.lib
    st = algo._env._stream()
    for grad, norm, p, m, v, step, lr, n in (
            (ts.grad_cbf, ts.norm_cbf, algo.cbf_params.flat, ts.m_cbf, ts.v_cbf, ts.step_cbf, algo.lr_cbf, ts.n_cbf),
            (ts.grad_act, ts.norm_act, algo.actor_net_params.flat, ts.m_act, ts.v_act, ts.step_act, algo.lr_actor,
             ts.n_act)):
        _lib.check(lib.gcbf_grad_sqnorm(_lib.ptr(grad), n, _lib.ptr(norm), st), "gcbf_grad_sqnorm")
        _lib.check(lib.gcbf_clip_adamw(_lib.ptr(p), _lib.ptr(grad), _lib.ptr(m), _lib.ptr(v), n, _lib.ptr(norm),
                                       _lib.ptr(step), lr, 0.9, 0.999, 1e-8, 1e-3, algo.max_grad_norm, st),
                   "gcbf_clip_adamw")


def read_info(algo) -> Dict[str, float]:
    """Info dict of the last minibatch with the reference's keys (gcbf_plus.py:423-440). Syncs."""
    ts: TrainState = algo._trainer_state
    if int(ts.overflow.item()) != 0:
        ts.overflow.zero_()
        raise RuntimeError("edge capacity overflow in a training / labelling graph: rows were dropped, the update is "
                           "invalid; raise env.edge_cap_per_agent")
    s = ts.stats.cpu().numpy().astype(np.float64)
    den = ts.denoms.cpu().numpy().astype(np.float64)
    n_unsafe, n_safe, n_tot = den[0], den[1], den[2]
    loss_unsafe = s[0] / (n_unsafe + 1e-6)
    loss_safe = s[1] / (n_safe + 1e-6)
    loss_h_dot = s[2] / n_tot
    loss_action = s[3] / n_tot
    total = (algo.loss_action_coef * loss_action + algo.loss_unsafe_coef * loss_unsafe +
             algo.loss_safe_coef * loss_safe + algo.loss_h_dot_coef * loss_h_dot)
    return {
        "grad_norm/cbf": float(np.sqrt(ts.norm_cbf[0].item())), "grad_norm/actor": float(np.sqrt(ts.norm_act[0].item())),
        "loss/action": loss_action, "loss/unsafe": loss_unsafe, "loss/safe": loss_safe, "loss/h_dot": loss_h_dot,
        "loss/total": total, "acc/unsafe": (s[4] + 1e-6) / (n_unsafe + 1e-6), "acc/safe": (s[5] + 1e-6) / (n_safe + 1e-6),
        "acc/h_dot": s[6] / n_tot, "acc/unsafe_data_ratio": n_unsafe / n_tot,
    }


def update_tgt(algo, tau: float = 0.5) -> None:
    """gcbf_plus.py:188-191,228."""
    env = algo._env
    _lib.check(env.lib.gcbf_polyak(_lib.ptr(algo.cbf_tgt_params.flat), _lib.ptr(algo.cbf_params.flat),
                                   algo.cbf_params.count, tau, env._stream()), "gcbf_polyak")


# ------------------------------------------------------------------------------------ labels
def label_rollout(algo, rollout: Rollout):
    """gcbf_plus.py:285-287: unsafe_mask of every stored graph (b, T) and the horizon safe mask.
    Returns uint8 tensors [b, T, N]."""
    env = algo._env
    lib = env.lib
    b, T, N = rollout.length, rollout.time_horizon, env.num_agents
    agent = rollout.agent[:, :T].reshape(b * T, N, env.state_dim).contiguous()
    hits = rollout.hits[:, :T].reshape(b * T, N, env.n_hits, env.pos_dim).contiguous()
    goal = rollout.goal[:, None].expand(b, T, N, env.state_dim).reshape(b * T, N, env.state_dim).contiguous()
    obs = rollout.obstacle
    O = obs.n_obs if obs is not None else 0
    packed = obs.packed[:, None].expand(b, T, *obs.packed.shape[1:]).reshape(b * T, *obs.packed.shape[1:]).contiguous() \
        if O > 0 else None
    d = env.desc(b * T, O, edge_cap=1)
    unsafe = torch.empty(b * T * N, dtype=torch.uint8, device=agent.device)
    _lib.check(lib.gcbf_masks(C.byref(d), _lib.ptr(agent), _lib.ptr(goal), _lib.ptr(hits), _lib.ptr(packed),
                              _lib.ptr(unsafe), None, None, None, env._stream()), "gcbf_masks")
    unsafe = unsafe.reshape(b, T, N)
    safe = torch.empty_like(unsafe)
    _lib.check(lib.gcbf_safe_horizon(_lib.ptr(unsafe), _lib.ptr(safe), b, T, N, algo.horizon, env._stream()),
               "gcbf_safe_horizon")
    return safe, unsafe


# ------------------------------------------------------------------------------------ update (gcbf_plus.py:282-297)
def _flatten_bt(rollout: Rollout, safe: torch.Tensor, unsafe: torch.Tensor):
    """(b, T, ...) -> dict of per-graph arrays [(b*T), ...]: the `merge01` of gcbf_plus.py:263-266."""
    b, T = rollout.length, rollout.time_horizon
    N = rollout.num_agents
    return {
        "agent": rollout.agent[:, :T].reshape(b * T, N, -1),
        "hits": rollout.hits[:, :T].reshape(b * T, N, *rollout.hits.shape[3:]),
        "goal": rollout.goal[:, None].expand(b, T, *rollout.goal.shape[1:]).reshape(b * T, N, -1),
        "safe": safe.reshape(b * T, N), "unsafe": unsafe.reshape(b * T, N),
    }


def _cat(parts):
    return {k: torch.cat([p[k] for p in parts], dim=0) for k in parts[0]}


def update(algo, rollout: Rollout, step: int) -> dict:
    """GCBFPlus.update (gcbf_plus.py:282-297) + sample_batch (:232-280) + update_nets (:198-230),
    with the replay kept on the device (SURVEY 8f2).  Action labels: the CBF-QP of every graph in the
    batch, solved on the device with the TARGET cbf (get_b_u_qp, :193-213) -- `batch_u_qp`."""
    env = algo._env
    require_one_layer(algo.cbf_params.n_layers, "update()")
    if algo._trainer_state is None:
        algo._trainer_state = TrainState(algo)
    if not hasattr(algo, "buffer"):
        algo.buffer = MaskedReplayBuffer(size=algo.buffer_size)
        algo.unsafe_buffer = MaskedReplayBuffer(size=algo.buffer_size // 2)
    safe, unsafe = label_rollout(algo, rollout)
    new = _flatten_bt(rollout, safe, unsafe)
    b, T = rollout.length, rollout.time_horizon
    if algo.buffer.length > algo.batch_size:
        memory = algo.buffer.sample_rollouts(b)                       # b stored rollouts -> b*T graphs
        unsafe_memory = algo.unsafe_buffer.sample_graphs(b * T) if algo.unsafe_buffer.length > 0 else memory
        algo.buffer.append_rollouts(new, b, T)
        algo.unsafe_buffer.append_graphs(new, new["unsafe"].any(dim=-1))
        batch = _cat([unsafe_memory, memory, new])
    else:
        algo.buffer.append_rollouts(new, b, T)
        algo.unsafe_buffer.append_graphs(new, new["unsafe"].any(dim=-1))
        batch = new
    n = batch["agent"].shape[0]
    qp_info: Dict[str, float] = {}
    u_qp = batch_u_qp(algo, batch, info=qp_info)
    # sharded run: this rank holds 1/world of the environments, so its share of every batch_size-graph minibatch
    # is batch_size / world graphs (same number of minibatches, hence of collectives, on every rank)
    dist = _dist()
    world = dist.get_world_size() if dist is not None else 1
    n_mb = max(n // max(algo.batch_size // world, 1), 1)
    mb_graphs = -(-n // n_mb)
    # exact upper bound on a minibatch's edge count from the per-graph counts measured while labelling: no
    # minibatch can overflow its edge lists whatever graphs the permutation puts together (ADVICE r1)
    mb_cap = max(int(qp_info["graph/max_edges"]) * mb_graphs, 64)
    # fixed-address copies of what the captured gather reads (the batch dict holds views / cat results of this update)
    batch = {k: v.contiguous() for k, v in batch.items()}
    bounds = np.concatenate([[0], np.cumsum([len(m) for m in np.array_split(np.arange(n), n_mb)])]).astype(np.int64)
    runners: Dict[int, MinibatchRunner] = {}
    for _ in range(algo.inner_epoch):
        idx = torch.from_numpy(algo.rng.permutation(n)).to(env.device)
        # label counts of all minibatches of the epoch: ONE small all-reduce per epoch instead of one per optimizer
        # step (the counts depend on the data only, SURVEY 8e)
        denoms_all = _minibatch_counts(batch, idx, bounds)
        if dist is not None:
            dist.all_reduce(denoms_all)
        for i in range(n_mb):
            lo, hi = int(bounds[i]), int(bounds[i + 1])
            r = runners.get(hi - lo)
            if r is None:
                r = runners[hi - lo] = MinibatchRunner(algo, batch, hi - lo, mb_cap, u_qp)
            r.run(idx[lo:hi], denoms_all[i])
    info = read_info(algo)
    info.update(qp_info)
    update_tgt(algo, 0.5)
    return info


def require_one_layer(n_layers: int, what: str) -> None:
    """The train step's backward and the QP labels' Lie-derivative Jacobian are one-hop (one GNN layer); deeper networks
    run forward only (rollouts, evaluation, h / pi)."""
    if n_layers != 1:
        raise NotImplementedError(f"{what} implements gnn_layers = 1, got {n_layers} GNN layers "
                                  "(forward, rollout and evaluation support any depth)")


def batch_u_ref(algo, batch) -> torch.Tensor:
    env = algo._env
    n = batch["agent"].shape[0]
    out = torch.empty(n, env.num_agents, env.action_dim, dtype=torch.float32, device=env.device)
    d = env.desc(n, 0, edge_cap=1)
    _lib.check(env.lib.gcbf_act(C.byref(d), _lib.ptr(batch["agent"].contiguous()), _lib.ptr(batch["goal"].contiguous()),
                                None, _lib.ptr(out), env._stream()), "gcbf_act")
    return out


# ------------------------------------------------------------------------------------ QP action labels
QP_MAX_ITER = 4000      # accelerated dual iterations per graph (early exit on QP_TOL; typical 50-1000)
QP_TOL = 1e-5           # projected dual-gradient residual


def qp_labels(algo, graph: SwarmGraph, params=None, with_aux: bool = False, max_iter: int = QP_MAX_ITER,
              tol: float = QP_TOL, with_iters: bool = False):
    """get_qp_action vmapped over the graphs of `graph` (gcbf_plus.py:193-196, 299-352): u_qp [G, N, nu];
    with_aux also returns (lam, r) [G, N, 2] and the iteration counts [G]; with_iters returns (u_qp, iters).
    A graph whose count equals max_iter stopped at the cap (its label is the capped iterate)."""
    env = algo._env
    lib = env.lib
    require_one_layer((params or algo.cbf_tgt_params).n_layers, "the CBF-QP labels")
    G, N = graph.n_graphs, env.num_agents
    d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
    cache = algo.__dict__.setdefault("_qp_ws", {})
    key = (G, d.edge_cap)
    if cache.get("key") != key:
        n = lib.gcbf_qp_workspace_floats(C.byref(d))
        if n <= 0:
            raise RuntimeError("gcbf_qp_workspace_floats failed")
        cache["ws"] = None
        cache["ws"] = torch.empty(int(n), dtype=torch.float32, device=env.device)
        cache["key"] = key
    ws = cache["ws"]
    p = params if params is not None else algo.cbf_tgt_params
    u_qp = torch.empty(G, N, env.action_dim, dtype=torch.float32, device=env.device)
    aux = torch.empty(G, N, 2, dtype=torch.float32, device=env.device) if with_aux else None
    iters = torch.empty(G, dtype=torch.int32, device=env.device) if (with_aux or with_iters) else None
    rc = lib.gcbf_qp_labels(C.byref(d), float(algo.alpha), 1 if _lib.USE_TC else 0, int(max_iter), float(tol),
                            _lib.ptr(p.flat), _lib.ptr(graph.agent), _lib.ptr(graph.goal), _lib.ptr(graph.hits),
                            _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_recv),
                            _lib.ptr(graph.edge_src), _lib.ptr(graph.counters), _lib.ptr(u_qp), _lib.ptr(aux),
                            _lib.ptr(iters), _lib.ptr(ws), ws.numel(), env._stream())
    _lib.check(rc, "gcbf_qp_labels")
    if with_aux:
        return u_qp, aux, iters & 0x3FFFFFFF      # bit 30 flags the global-memory fallback of dense graphs
    if with_iters:
        return u_qp, iters & 0x3FFFFFFF
    return u_qp


QP_POLISH_ITER = 60000   # second pass for the graphs that stopped at QP_MAX_ITER (same method, 15x the budget)


def batch_u_qp(algo, batch, agents_per_chunk: int = 32768, info: Optional[dict] = None) -> torch.Tensor:
    """update_nets' label pass (gcbf_plus.py:201-211): the reference cuts the batch into 8 chunks to bound the
    dense QP memory; here the chunk only bounds the activation workspace.

    No silent caps: every graph's iteration count is read back (one sync per update); graphs that stopped at
    QP_MAX_ITER are solved again with QP_POLISH_ITER, and what is still capped after that is reported
    (`qp/capped_frac` first pass, `qp/unconverged_frac` after the polish) in `info`.  The same pass measures the
    largest per-graph edge count (`graph/max_edges`, sizes the minibatch edge lists exactly) and ORs the
    edge-capacity overflow flags of the chunk graphs; an overflow doubles env.edge_cap_per_agent and relabels."""
    env = algo._env
    require_one_layer(algo.cbf_tgt_params.n_layers, "the CBF-QP labels")
    if algo._trainer_state is None:
        algo._trainer_state = TrainState(algo)
    ts: TrainState = algo._trainer_state
    n, N = batch["agent"].shape[0], env.num_agents
    chunk = max(1, agents_per_chunk // N)
    dev = env.device
    out = torch.empty(n, N, env.action_dim, dtype=torch.float32, device=dev)
    iters = torch.empty(n, dtype=torch.int32, device=dev)
    n_edges = torch.empty(n, dtype=torch.int32, device=dev)

    def sub_graph(sel):
        return env.get_graph(batch["agent"][sel].contiguous(), batch["goal"][sel].contiguous(), None,
                             hits=batch["hits"][sel].contiguous())

    for attempt in range(6):
        flag = torch.zeros(1, dtype=torch.int32, device=dev)
        for lo in range(0, n, chunk):
            hi = min(n, lo + chunk)
            g = sub_graph(slice(lo, hi))
            out[lo:hi], iters[lo:hi] = qp_labels(algo, g, with_iters=True)
            n_edges[lo:hi] = g.row_deg.reshape(hi - lo, N).sum(dim=1)
            flag |= g.counters[1:2]
        if int(flag.item()) == 0:                      # the one host sync of the label pass
            break
        env.edge_cap_per_agent *= 2                    # rows were dropped: grow the edge lists and label again
    else:
        raise RuntimeError("edge capacity overflow persists after growing env.edge_cap_per_agent 32x")
    capped = torch.nonzero(iters >= QP_MAX_ITER).flatten()
    n_capped = int(capped.numel())
    n_left = 0
    if n_capped:
        for lo in range(0, n_capped, chunk):
            sel = capped[lo:lo + chunk]
            g = sub_graph(sel)
            u2, it2 = qp_labels(algo, g, with_iters=True, max_iter=QP_POLISH_ITER)
            out[sel] = u2
            iters[sel] = it2
            ts.overflow |= g.counters[1:2]
        n_left = int((iters[capped] >= QP_POLISH_ITER).sum().item())
    if info is not None:
        info["qp/capped_frac"] = n_capped / n
        info["qp/unconverged_frac"] = n_left / n
        info["qp/iters_median"] = float(iters.float().median().item())
        info["graph/max_edges"] = int(n_edges.max().item())
        info["graph/mean_edges"] = float(n_edges.float().mean().item())
    return out
