#!/usr/bin/env python
"""Cost of observation and actuation noise in a GCBF+ actor rollout on one GPU (DESIGN.md 4.11).

    python tools/bench_noise.py [--config 3] [--T 64] [--rollouts 20] [--repeats 3]

Three rows at the shapes of bench.py's config (default: 3, the configs[2] shapes), each a whole T-step rollout replayed from one CUDA
graph with the reference's pretrained DoubleIntegrator actor (tests/golden): the noiseless actor on the persistent kernel
(where the configuration supports it), the noiseless actor on the step-by-step path (the fused gcbf_rollout_step_l), and
the perturbed actor (state, LiDAR and action noise; the modular sequence plus the two noise launches).  Prints one JSON
line: ms per rollout (every timed window: the spread), env-steps/s, launches per env-step, the slowdown of the perturbed
rollout against each noiseless one, and the card / power limit / clocks.  Writes nothing to the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import CONFIGS, metric_name  # noqa: E402
from bench_refine import _timed  # noqa: E402


def run(args) -> dict:
    import numpy as np
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.rollout import Perturbation, RolloutEngine
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_noise.py needs a CUDA device: the product path has no CPU fallback")
    _lib.load(build_if_missing=False)
    cfg = CONFIGS[args.config]
    env_id, N, T = cfg["env"], cfg["N"], args.T
    E = args.envs or max(cfg["envs_total"] // cfg["gpus"], 1)
    env = make_env(env_id, N, area_size=cfg["area"], num_obs=cfg["obs"], n_rays=cfg["rays"], device="cuda")
    algo = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, seed=0)
    algo.load_npz(os.path.join(ROOT, "tests", "golden", f"params_{env_id}.npz"))
    g0 = env.reset(1000, n_envs=E)
    pert = Perturbation(args.state_noise, args.lidar_noise, args.action_noise, seed=1234)
    out = {"metric": metric_name(cfg) + " policy=actor noise", "unit": "env-steps/s", "n_gpus": 1,
           "repeats": args.repeats,
           "config": {"workload": f"{env_id} n={N} envs={E} obs={cfg['obs']} n_rays={cfg['rays']} area={cfg['area']} "
                                  f"T={T} rollout ({cfg['name']} shapes)",
                      "sigmas": {"state": args.state_noise, "lidar": args.lidar_noise, "action": args.action_noise},
                      "gemm_path": "wgmma 3xTF32" if _lib.USE_TC else "strict-fp32 SIMT"}}
    clocks = []
    rows = (("persistent", dict(persistent=True)), ("step", dict(persistent=False)),
            ("perturbed", dict(perturbation=pert)))
    for name, kw in rows:
        try:
            eng = RolloutEngine(env, E, T=T, n_obs=cfg["obs"], **kw)
        except ValueError as e:       # the persistent kernel does not support this configuration
            out[name] = {"skipped": str(e)}
            continue
        eng.set_params(algo.actor_params)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        for _ in range(max(args.warmup, 1)):          # the first run captures the CUDA graph
            eng.run(check=False)
        torch.cuda.synchronize()
        ms = _timed(lambda: eng.run(check=False), args.rollouts, args.repeats, clocks)
        eng.check_overflow()
        med = float(np.median(ms))
        out[name] = {"value": N * E * T / (med * 1e-3), "ms_per_rollout": ms, "us_per_env_step": med / T * 1e3,
                     "launches_per_env_step": eng.launches_per_run / T}
        if name == "perturbed":
            out[name]["mean_abs_state_error"] = float((eng.obs_agent - eng.agent[:-1]).abs().mean())
        del eng
        torch.cuda.empty_cache()
    out["clocks"] = clocks
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    out["gpu"] = q.stdout.strip() if q.returncode == 0 else "unknown"
    out["value"] = out["perturbed"]["value"]
    for ref in ("persistent", "step"):
        if "value" in out[ref]:
            out[f"slowdown_vs_{ref}"] = out[ref]["value"] / out["perturbed"]["value"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3, choices=sorted(CONFIGS))
    ap.add_argument("--envs", type=int, default=None, help="default: the config's envs / its GPU count")
    ap.add_argument("--T", type=int, default=64)
    ap.add_argument("--rollouts", type=int, default=20, help="rollouts per timed window")
    ap.add_argument("--repeats", type=int, default=3, help="timed windows per row (the spread)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--state-noise", type=float, default=0.02)
    ap.add_argument("--lidar-noise", type=float, default=0.02)
    ap.add_argument("--action-noise", type=float, default=0.1)
    args = ap.parse_args()
    print(json.dumps(run(args)), flush=True)


if __name__ == "__main__":
    main()
