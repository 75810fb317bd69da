#!/usr/bin/env python
"""Throughput of the CBF-QP baseline rollouts (DecShareCBF / CentralizedCBF, csrc/cbfqp.cu) on one GPU.

    python tools/bench_cbfqp.py --policy dec_share_cbf [--config 3] [--steps 40] [--warmup 3]

Times the rollout leg of a bench.py workload (same configs, same seeded reset) with a baseline controller as the
policy: per env-step the pairwise CBFs + QP solve, env.step with the QP action, the graph build of the next state; the
whole rollout is one CUDA graph.  The baselines have no parameters, so there is no train leg.  Prints one JSON line:
env-steps/s, launches per env-step and the QP iteration statistics (median / max / capped) of the last timed rollout.
Writes nothing to the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import CONFIGS, T_STEPS, ClockSampler, metric_name  # noqa: E402


def run(args) -> dict:
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_cbfqp.py needs a CUDA device: the product path has no CPU fallback")
    _lib.load(build_if_missing=False)
    cfg = CONFIGS[args.config]
    env_id, N, T = cfg["env"], cfg["N"], args.T
    E = args.envs or max(cfg["envs_total"] // cfg["gpus"], 1)
    env = make_env(env_id, N, area_size=cfg["area"], num_obs=cfg["obs"], n_rays=cfg["rays"], device="cuda")
    g0 = env.reset(1000, n_envs=E)
    eng = RolloutEngine(env, E, T=T, n_obs=cfg["obs"], policy=args.policy)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    for _ in range(max(args.warmup, 3)):          # the first run captures the CUDA graph
        eng.run(check=False)
    torch.cuda.synchronize()
    eng.check_overflow()
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    sampler = ClockSampler(0)
    sampler.start()
    ev0.record()
    for _ in range(args.steps):
        eng.run(check=False)
    ev1.record()
    torch.cuda.synchronize()
    clocks = sampler.stop()
    eng.check_overflow()
    ms_per_step = ev0.elapsed_time(ev1) / args.steps
    ctl = eng.controller
    return {"metric": metric_name(cfg) + f" policy={args.policy}", "value": N * E * T / (ms_per_step * 1e-3),
            "unit": "env-steps/s", "n_gpus": 1, "steps": args.steps, "warmup": max(args.warmup, 3),
            "ms_per_step": ms_per_step, "higher_is_better": True, "policy": args.policy,
            "config": {"workload": f"{env_id} n={N} envs={E} obs={cfg['obs']} n_rays={cfg['rays']} area={cfg['area']} "
                                   f"T={T} rollout ({cfg['name']})", "step": f"one {T}-step rollout of {E} envs",
                       "alpha": ctl.alpha, "qp_max_iter": ctl.max_iter, "qp_tol": ctl.tol,
                       "us_per_env_step": ms_per_step / T * 1e3},
            "launches_per_env_step": eng.launches_per_run / T,
            "gpu_launches": eng.launches_per_run * args.steps,
            "qp": eng.qp_stats(),                # every solve of the last timed rollout
            "clocks": clocks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--policy", type=str, required=True, choices=["dec_share_cbf", "centralized_cbf"])
    ap.add_argument("--config", type=int, default=3, choices=sorted(CONFIGS))
    ap.add_argument("--envs", type=int, default=None, help="default: the config's envs / its GPU count")
    ap.add_argument("--steps", type=int, default=40)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--T", type=int, default=T_STEPS)
    print(json.dumps(run(ap.parse_args())))


if __name__ == "__main__":
    main()
