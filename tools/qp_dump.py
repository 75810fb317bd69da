#!/usr/bin/env python
"""Outputs of the four device QP entry points on seeded inputs, and a byte-for-byte comparison of two such dumps.

    python tools/qp_dump.py OUT_DIR
    python tools/qp_dump.py --compare DIR_A DIR_B

Calls gcbf_qp_labels, gcbf_qp_filter, gcbf_cbfqp_dec_share and gcbf_cbfqp_centralized directly and writes u, aux / r
and iters of every case as .npy files, with index.json listing them.  The cases:
  * all four environments at N = 8, 64 and 512 (pretrained CBF from tests/golden, random scenes with obstacles);
  * the labels and the filter on both dense-layer paths (use_tensor_cores 0 and 1);
  * filter nominals u_ref + noise of 2 u_lim, so that components lie outside the box;
  * max_iter = 3 at N = 64: the capped iterate;
  * agent 0 of graph 0 exactly at its goal (u_ref is NaN there, except for DubinsCar) at N = 8;
  * the labels' dense-graph fallback: 64 DoubleIntegrator agents that all neighbour each other.
Run it on two builds on the same GPU model; --compare exits non-zero unless every array is byte-identical."""
import argparse
import ctypes as C
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))


def _scene(env_id, N, G, area, n_obs, seed, at_goal=False, edge_cap_per_agent=64):
    import torch
    from helpers import product_algo, product_env, product_obstacles, random_scene
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed)
    if at_goal:
        agent[0, 0] = goal[0, 0]
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = edge_cap_per_agent
    algo = product_algo(env, env_id)
    pobs = product_obstacles(env_id, obs) if n_obs else None
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    return env, algo, graph


def _labels(env, algo, graph, use_tc, max_iter, tol, u_nom=None):
    """gcbf_qp_labels (u_nom None) or gcbf_qp_filter: u, aux, iters (raw words)."""
    import torch
    from gcbfplus_b200 import _lib
    G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
    d = env.desc(G, 0, edge_cap=graph.edge_recv.numel())
    ws = torch.empty(int(env.lib.gcbf_qp_workspace_floats(C.byref(d))), dtype=torch.float32, device="cuda")
    u = torch.empty(G, N, nu, dtype=torch.float32, device="cuda")
    aux = torch.empty(G, N, 2, dtype=torch.float32, device="cuda")
    iters = torch.empty(G, dtype=torch.int32, device="cuda")
    head = (C.byref(d), float(algo.alpha), int(use_tc), int(max_iter), float(tol), _lib.ptr(algo.cbf_params.flat),
            _lib.ptr(graph.agent), _lib.ptr(graph.goal), _lib.ptr(graph.hits), _lib.ptr(graph.row_start),
            _lib.ptr(graph.row_deg), _lib.ptr(graph.edge_recv), _lib.ptr(graph.edge_src), _lib.ptr(graph.counters))
    tail = (_lib.ptr(u), _lib.ptr(aux), _lib.ptr(iters), _lib.ptr(ws), ws.numel(), env._stream())
    if u_nom is None:
        _lib.check(env.lib.gcbf_qp_labels(*head, *tail), "gcbf_qp_labels")
    else:
        _lib.check(env.lib.gcbf_qp_filter(*head, _lib.ptr(u_nom), *tail), "gcbf_qp_filter")
    return {"u": u, "aux": aux, "iters": iters}


def _baseline(env, graph, entry, max_iter, tol, alpha=1.0):
    """gcbf_cbfqp_dec_share / gcbf_cbfqp_centralized: u, r, iters (raw words)."""
    import torch
    from gcbfplus_b200 import _lib
    G, N, nu = graph.n_graphs, env.num_agents, env.action_dim
    d = env.desc(G, 0, edge_cap=1)
    ws = torch.empty(max(int(env.lib.gcbf_cbfqp_workspace_floats(C.byref(d))), 1), dtype=torch.float32, device="cuda")
    u = torch.empty(G, N, nu, dtype=torch.float32, device="cuda")
    r = torch.empty(G, N, 3, dtype=torch.float32, device="cuda")
    iters = torch.empty(G * N if entry == "gcbf_cbfqp_dec_share" else G, dtype=torch.int32, device="cuda")
    rc = getattr(env.lib, entry)(C.byref(d), float(alpha), int(max_iter), float(tol), _lib.ptr(graph.agent),
                                 _lib.ptr(graph.goal), _lib.ptr(graph.hits), _lib.ptr(u), _lib.ptr(r), _lib.ptr(iters),
                                 _lib.ptr(ws), ws.numel(), env._stream())
    _lib.check(rc, entry)
    return {"u": u, "r": r, "iters": iters}


def dump(out_dir: str) -> None:
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo.cbf_qp import QP_MAX_ITER as CBF_MAX_ITER, QP_TOL as CBF_TOL
    from gcbfplus_b200.algo.train import QP_MAX_ITER, QP_TOL
    from helpers import ENVS
    if not torch.cuda.is_available():
        raise RuntimeError("tools/qp_dump.py needs a CUDA device")
    _lib.load(build_if_missing=False)
    os.makedirs(out_dir, exist_ok=True)
    index = {}

    def save(case, arrays):
        torch.cuda.synchronize()
        for k, v in arrays.items():
            name = f"{case}.{k}"
            a = v.cpu().numpy()
            np.save(os.path.join(out_dir, name + ".npy"), a)
            index[name] = {"shape": list(a.shape), "dtype": str(a.dtype)}

    def run_case(tag, env, algo, graph, max_iter=None, baselines=True):
        graph.check_overflow()
        rng = np.random.default_rng(5)
        u_ref = env.u_ref(graph)
        u_nom = (u_ref + torch.from_numpy(rng.normal(size=tuple(u_ref.shape)).astype(np.float32)).cuda()
                 * (2.0 * float(env.action_lim()[1][0]))).contiguous()
        for tc in (0, 1):
            save(f"{tag}.labels.tc{tc}", _labels(env, algo, graph, tc, max_iter or QP_MAX_ITER, QP_TOL))
            save(f"{tag}.filter.tc{tc}", _labels(env, algo, graph, tc, max_iter or QP_MAX_ITER, QP_TOL, u_nom))
        if baselines:
            for entry in ("gcbf_cbfqp_dec_share", "gcbf_cbfqp_centralized"):
                save(f"{tag}.{entry[11:]}", _baseline(env, graph, entry, max_iter or CBF_MAX_ITER, CBF_TOL))

    for env_id in ENVS:
        dim = 3 if env_id == "LinearDrone" else 2
        for N in (8, 64, 512):
            G = 4 if N <= 64 else 2
            area = (0.8 if env_id == "LinearDrone" else 1.5) * (N / 8) ** (1 / dim)
            env, algo, graph = _scene(env_id, N, G, area, 4, seed=300 + N)
            run_case(f"{env_id}.N{N}", env, algo, graph)
            if N == 64:
                run_case(f"{env_id}.N{N}.cap3", env, algo, graph, max_iter=3)
            if N == 8:
                env, algo, graph = _scene(env_id, N, G, area, 4, seed=300 + N, at_goal=True)
                run_case(f"{env_id}.N{N}.at_goal", env, algo, graph)
    # the scene of tests/test_gpu_qp.py::test_qp_labels_dense_graph_fallback (63 blocks per row > 24 in shared memory)
    import helpers
    agent, goal, _ = helpers.random_scene("DoubleIntegrator", 64, 2, 0.3, 0, seed=8)
    goal[..., :2] += 1.0
    env = helpers.product_env("DoubleIntegrator", 64, 0.3, 0)
    env.edge_cap_per_agent = 128
    algo = helpers.product_algo(env, "DoubleIntegrator")
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), None)
    run_case("dense_fallback", env, algo, graph, baselines=False)
    dense = int((_lib.split_iters(np.load(os.path.join(out_dir, "dense_fallback.labels.tc0.iters.npy")))[1]).sum())
    assert dense == 2, f"the dense scene took the shared-memory path in {2 - dense} of 2 graphs"
    with open(os.path.join(out_dir, "index.json"), "w") as f:
        json.dump(index, f, indent=1, sort_keys=True)
    print(json.dumps({"arrays": len(index), "out": out_dir}))


def compare(a_dir: str, b_dir: str) -> int:
    ia = json.load(open(os.path.join(a_dir, "index.json")))
    ib = json.load(open(os.path.join(b_dir, "index.json")))
    bad = sorted(set(ia) ^ set(ib))
    for name in sorted(set(ia) & set(ib)):
        a = np.load(os.path.join(a_dir, name + ".npy"))
        b = np.load(os.path.join(b_dir, name + ".npy"))
        same = a.dtype == b.dtype and a.shape == b.shape and a.tobytes() == b.tobytes()
        print(f"{'same' if same else 'DIFF'} {name}")
        if not same:
            bad.append(name)
    print(json.dumps({"arrays": len(set(ia) | set(ib)), "identical": not bad, "differ": bad}))
    return 1 if bad else 0


if __name__ == "__main__":
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("out", nargs="?")
    ap.add_argument("--compare", nargs=2, metavar=("DIR_A", "DIR_B"))
    args = ap.parse_args()
    if args.compare:
        sys.exit(compare(*args.compare))
    if not args.out:
        ap.error("give OUT_DIR or --compare DIR_A DIR_B")
    dump(args.out)
