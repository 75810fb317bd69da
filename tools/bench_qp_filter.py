#!/usr/bin/env python
"""Cost of the learned-CBF QP safety filter in a rollout (the rollout engine's actor_qp / u_ref_qp policies) on one
GPU, next to the plain actor and online policy refinement (actor_refine) on the same step-by-step path.

    python tools/bench_qp_filter.py [--T 64] [--repeats 3] [--sizes 512,64]

Per env-step the filter policies run the nominal action (actor_qp: actor forward + 2 pi + u_ref; u_ref_qp: u_ref),
gcbf_qp_filter (CBF forward, data-only backward for the Jacobian, QP assembly, one CTA per graph for the dual solve)
and env.step + canonical graph build; the whole rollout is one CUDA graph for every policy.  The workload is
DoubleIntegrator with 16 environments, 8 obstacles and 32 rays: n = 512 on configs[2]'s 32 x 32 area, and each smaller
n on an area scaled to the same agent density.  The reference's pretrained networks (tests/golden) are used.
Each timed window runs every policy in turn (`--rollouts` whole rollouts each), so the policies alternate over the
`--repeats` windows.  Prints one JSON line per size: ms per rollout per window, us per env-step, env-steps/s, launches
per env-step, the solver's iteration statistics of the last timed rollout, and the card, its power limit and the clocks
sampled over the timed windows.  Writes nothing to the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import CONFIGS, ClockSampler  # noqa: E402

POLICIES = ("actor", "actor_refine", "actor_qp", "u_ref_qp")


def _gpu() -> str:
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    return q.stdout.strip() if q.returncode == 0 else "unknown"


def run(args, N: int) -> dict:
    import numpy as np
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.algo.train import QP_MAX_ITER, QP_TOL
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_qp_filter.py needs a CUDA device: the product path has no CPU fallback")
    _lib.load(build_if_missing=False)
    cfg = CONFIGS[3]
    env_id, E, T = cfg["env"], args.envs, args.T
    area = cfg["area"] * float(np.sqrt(N / cfg["N"]))
    env = make_env(env_id, N, area_size=area, num_obs=cfg["obs"], n_rays=cfg["rays"], device="cuda")
    algo = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, seed=0)
    algo.load_npz(os.path.join(ROOT, "tests", "golden", f"params_{env_id}.npz"))
    g0 = env.reset(1000, n_envs=E)
    engines = {}
    for policy in POLICIES:
        eng = RolloutEngine(env, E, T=T, n_obs=cfg["obs"], policy=policy, persistent=False)
        eng.set_params(algo.actor_params)
        if policy != "actor":
            eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        for _ in range(max(args.warmup, 1)):          # the first run captures the CUDA graph
            eng.run(check=False)
        engines[policy] = eng
    torch.cuda.synchronize()
    n_runs = dict(zip(POLICIES, args.rollouts))
    ms = {p: [] for p in POLICIES}
    sampler = ClockSampler(0)
    sampler.start()
    try:
        for _ in range(args.repeats):
            for policy in POLICIES:
                eng = engines[policy]
                ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                ev0.record()
                for _ in range(n_runs[policy]):
                    eng.run(check=False)
                ev1.record()
                torch.cuda.synchronize()
                ms[policy].append(ev0.elapsed_time(ev1) / n_runs[policy])
    finally:
        clocks = sampler.stop()
    out = {"metric": f"ms per {T}-step rollout, {env_id} n={N} envs={E}", "n_gpus": 1, "repeats": args.repeats,
           "config": {"workload": f"{env_id} n={N} envs={E} obs={cfg['obs']} n_rays={cfg['rays']} area={area:.2f} T={T}",
                      "weights": "pretrained (tests/golden)", "qp_max_iter": QP_MAX_ITER, "qp_tol": QP_TOL,
                      "gemm_path": "wgmma 3xTF32" if _lib.USE_TC else "strict-fp32 SIMT"}}
    for policy in POLICIES:
        eng = engines[policy]
        eng.check_overflow()
        med = float(np.median(ms[policy]))
        row = {"ms_per_rollout": ms[policy], "rollouts_per_window": n_runs[policy], "us_per_env_step": med / T * 1e3,
               "env_steps_per_s": N * E * T / (med * 1e-3), "launches_per_env_step": eng.launches_per_run / T,
               "vs_actor": med / float(np.median(ms["actor"]))}
        if policy == "actor_refine":
            row["refine"] = eng.refine_stats()
        elif policy != "actor":
            it, dense = _lib.split_iters(eng.chains[0].qp_iters.reshape(-1).to(torch.int64).cpu().numpy())
            row["qp"] = dict(eng.qp_stats(), iters_mean=float(it.mean()),
                             iters_p90=float(np.percentile(it, 90)), iters_p99=float(np.percentile(it, 99)),
                             dense_fallback=int(dense.sum()))
        out[policy] = row
    out["clocks"] = clocks
    out["gpu"] = _gpu()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", type=str, default="512,64", help="agent counts n, comma-separated")
    ap.add_argument("--envs", type=int, default=16)
    ap.add_argument("--T", type=int, default=64)
    ap.add_argument("--rollouts", type=str, default="20,1,2,2",
                    help="rollouts per timed window of " + ", ".join(POLICIES))
    ap.add_argument("--repeats", type=int, default=3, help="timed windows (the spread)")
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    args.rollouts = [int(x) for x in args.rollouts.split(",")]
    if len(args.rollouts) != len(POLICIES):
        ap.error(f"--rollouts takes {len(POLICIES)} counts")
    for n in (int(x) for x in args.sizes.split(",")):
        print(json.dumps(run(args, n)), flush=True)


if __name__ == "__main__":
    main()
