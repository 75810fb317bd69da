"""Rollout throughput and CBF forward device time for GNN depth L = 1 and L = 2 (--gnn-layers) at BASELINE.json configs[2]
shapes (DoubleIntegrator, n = 512, 16 environments, 8 obstacles, 32 rays), both depths on the step-by-step CUDA-graph
rollout path.  Prints one JSON line with the GPU name and power limit.  Networks are xavier-initialised (the timing does
not depend on the weights).  The train step and the QP labels implement L = 1 only and are not measured here.

    python tools/bench_gnn_layers.py [--steps 5] [--T 256]
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    name, _, power = q.stdout.strip().splitlines()[0].partition(",") if q.returncode == 0 else ("unknown", "", "unknown")
    return name.strip(), power.strip()


def cbf_forward_device_ms(env, params, graph, reps: int = 20) -> float:
    import ctypes as C
    from gcbfplus_b200 import _lib
    dev = graph.agent.device
    d = env.desc(graph.n_graphs, 0, edge_cap=graph.edge_recv.numel())
    pt = params.prepared()
    n_ws = env.lib.gcbf_gnn_workspace_floats_l(C.byref(d), 1, params.n_layers)
    ws = torch.empty(int(n_ws), dtype=torch.float32, device=dev)
    out = torch.empty(graph.n_graphs, env.num_agents, 1, dtype=torch.float32, device=dev)

    def fwd():
        _lib.check(env.lib.gcbf_gnn_forward_l(
            C.byref(d), _lib.NET_CBF, 1, params.n_layers, _lib.ptr(params.flat), _lib.ptr(pt), _lib.ptr(graph.agent),
            _lib.ptr(graph.goal), _lib.ptr(graph.hits), _lib.ptr(graph.row_start), _lib.ptr(graph.row_deg),
            _lib.ptr(graph.edge_recv), _lib.ptr(graph.edge_src), _lib.ptr(graph.counters), 0, _lib.ptr(out),
            _lib.ptr(ws), ws.numel(), torch.cuda.current_stream(dev).cuda_stream), "gcbf_gnn_forward_l")

    fwd()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(reps):
            fwd()
    g.replay()
    torch.cuda.synchronize()
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(5):
        g.replay()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / (5 * reps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5, help="timed rollouts per depth")
    ap.add_argument("--T", type=int, default=256, help="env steps per rollout")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise RuntimeError("bench_gnn_layers.py needs a CUDA device")
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    N, E, n_obs, area = 512, 16, 8, 32.0      # bench.py CONFIGS[3] (BASELINE configs[2])
    env = make_env("DoubleIntegrator", N, area_size=area, num_obs=n_obs, n_rays=32)
    g0 = env.reset(1000, n_envs=E)
    out = {"gpu": None, "power_limit": None, "config": f"DoubleIntegrator n={N}, {E} envs, obs {n_obs}, T={args.T}"}
    out["gpu"], out["power_limit"] = gpu_info()
    for L in (1, 2):
        algo = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                         action_dim=env.action_dim, n_agents=N, gnn_layers=L, seed=0)
        eng = RolloutEngine(env, E, T=args.T, n_obs=n_obs, persistent=False)
        eng.set_params(algo.actor_params)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        for _ in range(3):
            eng.run(check=False)
        torch.cuda.synchronize()
        eng.check_overflow()
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(args.steps):
            eng.run(check=False)
        t1.record()
        torch.cuda.synchronize()
        ms = t0.elapsed_time(t1) / args.steps
        # one CBF forward over the graphs of the last rollout step, device time only: the weight planes are prepared
        # once and 20 forwards are captured in one CUDA graph, so neither the plane rebuild of GnnRunner.forward nor
        # host dispatch is in the window
        graph = env.get_graph(eng.agent[-1].contiguous(), eng.goal, g0.obstacle)
        fwd_ms = cbf_forward_device_ms(env, algo.cbf_params, graph)
        out[f"L{L}"] = {"rollout_ms": round(ms, 3), "env_steps_per_s": round(E * N * args.T / (ms * 1e-3)),
                        "launches_per_rollout": eng.launches_per_run, "cbf_forward_device_ms": round(fwd_ms, 4),
                        "forward_edges": int(graph.counters[0])}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
