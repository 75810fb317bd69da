#!/usr/bin/env python
"""Cost of the CBF falsification search (GCBFPlus.falsify) on one GPU.

    python tools/bench_falsify.py [--iters 20] [--calls 20] [--repeats 3]

Two shapes of the DoubleIntegrator with the reference's pretrained networks (tests/golden/params_DoubleIntegrator.npz):
16 graphs x 512 agents with 8 obstacles, and 1024 graphs x 8 agents.  Per shape, from CUDA events:
  condition      ms per gcbf_cbf_condition call without the gradient (3 forwards + selection)
  condition_grad ms per call with the gradient (+ 3 data-only backwards and the chain kernels)
  search         ms per iteration of falsify(--iters): graph build + condition_grad + the step, host syncs included
Every row is --repeats timed windows (the spread).  Prints one JSON line per shape with the card name, power limit and
maximum SM clock read in the same run.  Writes nothing to the tree."""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [("DoubleIntegrator", 16, 512, 8), ("DoubleIntegrator", 1024, 8, 0)]


def _timed(fn, n: int, repeats: int) -> list:
    import torch
    out = []
    for _ in range(repeats):
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record()
        for _ in range(n):
            fn()
        ev1.record()
        torch.cuda.synchronize()
        out.append(ev0.elapsed_time(ev1) / n)
    return out


def run(args, env_id: str, G: int, N: int, n_obs: int) -> dict:
    import numpy as np
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.algo.falsify import CbfCondition
    from gcbfplus_b200.env import make_env
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_falsify.py needs a CUDA device: the product path has no CPU fallback")
    _lib.load(build_if_missing=False)
    area = float(np.sqrt(N)) * 0.5 + 1.0            # about 4 agents per unit area: neighbours in the radius graph
    env = make_env(env_id, N, area_size=area, num_obs=n_obs, device="cuda")
    env.edge_cap_per_agent = 64
    algo = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, seed=0)
    algo.load_npz(os.path.join(ROOT, "tests", "golden", f"params_{env_id}.npz"))
    g0 = env.reset(1000, n_envs=G)
    graph = env.get_graph(g0.agent, g0.goal, g0.obstacle)
    cond = CbfCondition(algo)
    out = {"metric": f"falsify {env_id} graphs={G} agents={N} obs={n_obs}", "unit": "ms",
           "gemm_path": "wgmma 3xTF32" if _lib.USE_TC else "strict-fp32 SIMT", "repeats": args.repeats}
    for name, grad in (("condition", False), ("condition_grad", True)):
        cond(graph, with_grad=grad)
        torch.cuda.synchronize()
        out[name] = {"ms_per_call": _timed(lambda: cond(graph, with_grad=grad), args.calls, args.repeats)}
    graph.check_overflow()
    algo.falsify(g0.agent, g0.goal, g0.obstacle, 2)                   # warm-up: workspaces, edge capacity
    torch.cuda.synchronize()
    ms = _timed(lambda: algo.falsify(g0.agent, g0.goal, g0.obstacle, args.iters), 1, args.repeats)
    r = algo.falsify(g0.agent, g0.goal, g0.obstacle, args.iters)
    out["search"] = {"ms_per_iteration": [m / args.iters for m in ms], "iters": args.iters,
                     "violating_start": float((r["J0"] > 0).float().mean()),
                     "violating_found": float((r["J"] > 0).float().mean())}
    out["value"] = float(np.median(out["search"]["ms_per_iteration"]))
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    out["gpu"] = q.stdout.strip() if q.returncode == 0 else "unknown"
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20, help="search iterations per timed falsify call")
    ap.add_argument("--calls", type=int, default=20, help="gcbf_cbf_condition calls per timed window")
    ap.add_argument("--repeats", type=int, default=3, help="timed windows per row (the spread)")
    args = ap.parse_args()
    for shape in SHAPES:
        print(json.dumps(run(args, *shape)), flush=True)


if __name__ == "__main__":
    main()
