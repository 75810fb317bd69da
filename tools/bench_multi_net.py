#!/usr/bin/env python
"""Evaluating K actor networks: K solo persistent rollout launches against one K-network launch
(gcbf_rollout_persistent_multi, RolloutEngine(n_nets=K)) on one GPU.

    python tools/bench_multi_net.py [--sizes 8,64] [--nets 1,4,16,64] [--epi 32] [--T 256] [--repeats 3]

The workload is the reference's evaluation setting: DoubleIntegrator, 8 obstacles, 32 rays, `--epi` episodes per
network, T env-steps; n = 8 on a 4 x 4 area and each larger n on an area scaled to the same agent density.  The networks
are xavier-initialised with seeds 0..K-1.  Every engine (the K solo ones, one per network, and the batched one) is
captured as a CUDA graph before the timed windows; each window replays the K solo rollouts back to back, then the
batched rollout, so the two alternate over `--repeats` windows (device events around each).  Also reported: whether the
batched launch's clusters are all co-resident (gcbf_rollout_persistent_supported: 2 = yes, 1 = the launch runs in
rounds), the co-resident cluster count, whether every network's record equals its solo record bit for bit, and the card
and its power limit read in the same run.  Prints one JSON line per (n, K).  Writes nothing to the tree."""
import argparse
import ctypes as C
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu() -> str:
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def run(args, N: int, K: int) -> dict:
    import numpy as np
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo.params import NetParams
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_multi_net.py needs a CUDA device: the product path has no CPU fallback")
    lib = _lib.load(build_if_missing=False)
    area = 4.0 * float(np.sqrt(N / 8))
    B, T, O = args.epi, args.T, 8
    env = make_env("DoubleIntegrator", N, area_size=area, num_obs=O, n_rays=32, device="cuda")
    nets = [NetParams(env.edge_dim, env.action_dim, "actor").init_xavier(s) for s in range(K)]
    g0 = env.reset(1000, n_envs=B)
    solo = []
    for p in nets:
        eng = RolloutEngine(env, B, T=T, n_obs=O, persistent=True)
        eng.set_params(p)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        eng.run(check=False)                           # captures the CUDA graph
        solo.append(eng)
    multi = RolloutEngine(env, K * B, T=T, n_obs=O, persistent=True, n_nets=K)
    multi.set_params(nets)
    obstacle = g0.obstacle.repeat(K)
    multi.set_initial(g0.agent.repeat(K, 1, 1), g0.goal.repeat(K, 1, 1), obstacle)
    multi.run(check=False)
    torch.cuda.synchronize()
    ms = {"solo": [], "multi": []}
    for _ in range(args.repeats):
        for name, engines in (("solo", solo), ("multi", [multi])):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for eng in engines:
                eng.run(check=False)
            ev1.record()
            torch.cuda.synchronize()
            ms[name].append(ev0.elapsed_time(ev1))
    for eng in solo + [multi]:
        eng.check_overflow()
    identical = all(torch.equal(multi.agent[:, idx], s.agent) and torch.equal(multi.actions[:, idx], s.actions)
                    and torch.equal(multi.rewards[:, idx], s.rewards) and torch.equal(multi.net_counters(k), s.counters)
                    for k, (idx, s) in enumerate(zip(multi.net_envs, solo)))
    level = int(lib.gcbf_rollout_persistent_supported(C.byref(multi._pdesc)))
    solo_med, multi_med = float(np.median(ms["solo"])), float(np.median(ms["multi"]))
    return {"metric": f"ms to roll out {K} networks x {B} episodes, DoubleIntegrator n={N}",
            "config": {"workload": f"DoubleIntegrator n={N} area={area:.2f} obs={O} n_rays=32 T={T}",
                       "networks": K, "episodes_per_network": B, "weights": "xavier, seeds 0..K-1"},
            "solo_ms": ms["solo"], "multi_ms": ms["multi"], "solo_over_multi": solo_med / multi_med,
            "batched_supported": level, "batched_clusters": K * B,
            "resident_clusters_of_2": int(lib.gcbf_rollout_persistent_max_clusters(2)), "bit_identical": bool(identical),
            "repeats": args.repeats, "gpu": _gpu()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="8,64", help="agent counts n, comma-separated")
    ap.add_argument("--nets", type=str, default="1,4,16,64", help="network counts K, comma-separated")
    ap.add_argument("--epi", type=int, default=32, help="episodes per network")
    ap.add_argument("--T", type=int, default=256)
    ap.add_argument("--repeats", type=int, default=3, help="timed windows (the spread)")
    args = ap.parse_args()
    for n in (int(x) for x in args.sizes.split(",")):
        for k in (int(x) for x in args.nets.split(",")):
            print(json.dumps(run(args, n, k)), flush=True)


if __name__ == "__main__":
    main()
