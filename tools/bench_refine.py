#!/usr/bin/env python
"""Throughput of GCBF+ rollouts with online policy refinement (the rollout engine's actor_refine policy) on one GPU,
next to the plain actor on the same step-by-step path.

    python tools/bench_refine.py [--config 3] [--T 64] [--steps 2] [--actor-rollouts 100] [--repeats 3]

Per env-step the refined policy runs the actor forward, gcbf_refine_actions (h, h(g'(u_ref)), then up to 30 iterations
of forward + value + data-only backward + update, gcbf.py:161-201) and env.step + graph build; the whole rollout is one
CUDA graph.  Both weight sets are measured: the reference's pretrained DoubleIntegrator networks
(tests/golden/params_DoubleIntegrator.npz) and xavier-initialised ones.  Prints one JSON line per weight set:
env-steps/s of actor_refine and of actor (step path, persistent kernel off), launches per env-step, the distribution
of refinement iterations per graph-step, the capped fraction, and the card / power limit / clocks (sampled over the timed windows).  Every row is
`--repeats` timed windows (the spread).  The early-exit row times GCBFPlus.online_policy_refinement on one batch at the
same shapes where every graph stops at iteration 1, with max_iter = 30 against max_iter = 1: the cost of an iteration
that runs after every graph has stopped.  Writes nothing to the tree."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import CONFIGS, metric_name  # noqa: E402


def _timed(fn, n: int, repeats: int, sampler_box: list) -> list:
    """ms per call of fn() over `repeats` windows of n calls each (CUDA events); the clock sampler runs over the timed
    windows only."""
    import torch
    from bench import ClockSampler
    out = []
    sampler = ClockSampler(0)
    sampler.start()
    try:
        for _ in range(repeats):
            ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            ev0.record()
            for _ in range(n):
                fn()
            ev1.record()
            torch.cuda.synchronize()
            out.append(ev0.elapsed_time(ev1) / n)
    finally:
        sampler_box.append(sampler.stop())
    return out


def run(args, weights: str) -> dict:
    import numpy as np
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_refine.py needs a CUDA device: the product path has no CPU fallback")
    _lib.load(build_if_missing=False)
    cfg = CONFIGS[args.config]
    env_id, N, T = cfg["env"], cfg["N"], args.T
    E = args.envs or max(cfg["envs_total"] // cfg["gpus"], 1)
    env = make_env(env_id, N, area_size=cfg["area"], num_obs=cfg["obs"], n_rays=cfg["rays"], device="cuda")
    algo = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, seed=0)
    if weights == "pretrained":
        algo.load_npz(os.path.join(ROOT, "tests", "golden", f"params_{env_id}.npz"))
    g0 = env.reset(1000, n_envs=E)
    out = {"metric": metric_name(cfg) + f" policy=actor_refine weights={weights}", "unit": "env-steps/s",
           "n_gpus": 1, "repeats": args.repeats, "weights": weights,
           "config": {"workload": f"{env_id} n={N} envs={E} obs={cfg['obs']} n_rays={cfg['rays']} area={cfg['area']} "
                                  f"T={T} rollout ({cfg['name']} shapes)", "refine_lr": 0.1, "refine_max_iter": 30,
                      "gemm_path": "wgmma 3xTF32" if _lib.USE_TC else "strict-fp32 SIMT"}}
    clocks = []
    # ---- rollouts on the step path: the plain actor and the refined policy (each window: `n` whole rollouts)
    for policy, n in (("actor", args.actor_rollouts), ("actor_refine", args.steps)):
        eng = RolloutEngine(env, E, T=T, n_obs=cfg["obs"], policy=policy, persistent=False)
        eng.set_params(algo.actor_params)
        if policy == "actor_refine":
            eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
        eng.set_initial(g0.agent, g0.goal, g0.obstacle)
        for _ in range(max(args.warmup, 1)):          # the first run captures the CUDA graph
            eng.run(check=False)
        torch.cuda.synchronize()
        ms = _timed(lambda: eng.run(check=False), n, args.repeats, clocks)
        eng.check_overflow()
        med = float(np.median(ms))
        out[policy] = {"value": N * E * T / (med * 1e-3), "ms_per_rollout": ms, "us_per_env_step": med / T * 1e3,
                       "rollouts_per_window": n, "launches_per_env_step": eng.launches_per_run / T}
        if policy == "actor_refine":
            it = eng.chains[0].refine_iters.reshape(-1).to(torch.int64).cpu().numpy()   # last timed rollout
            k, capped = _lib.split_iters(it)
            out["refine"] = dict(eng.refine_stats(), capped_frac=float(capped.mean()),
                                 iters_mean=float(k.mean()),
                                 iters_hist={int(a): int(b) for a, b in zip(*np.unique(k, return_counts=True))})
        del eng
        torch.cuda.empty_cache()
    if weights != "pretrained":     # a random CBF is not positive on a spread-out scene: no graph would stop early
        return _finish(out, clocks)
    # ---- the early exit: one batch of E graphs at the same shapes whose loop value is 0 at iteration 1 -- drawn from a
    # pool of spread-out scenes (no neighbours, no obstacles, at rest, goals nearby), keeping the graphs that stop there;
    # max_iter = 30 against max_iter = 1 gives the cost of the 29 iterations that run with zero row counts
    rng = np.random.default_rng(7)
    sd, pool = env.state_dim, 4 * E
    side = float(np.sqrt(64.0 * N))
    ag = np.zeros((pool, N, sd), np.float32)
    gl = np.zeros((pool, N, sd), np.float32)
    ag[..., :2] = rng.uniform(0, side, size=(pool, N, 2))
    gl[..., :2] = ag[..., :2] + rng.uniform(-0.3, 0.3, size=(pool, N, 2))
    senv = make_env(env_id, N, area_size=side, num_obs=0, n_rays=cfg["rays"], device="cuda")
    salgo = make_algo("gcbf+", env=senv, node_dim=senv.node_dim, edge_dim=senv.edge_dim, state_dim=sd,
                      action_dim=senv.action_dim, n_agents=N, seed=0)
    salgo.cbf_params.flat.copy_(algo.cbf_params.flat)
    salgo.actor_net_params.flat.copy_(algo.actor_net_params.flat)
    graph = senv.get_graph(torch.from_numpy(ag).cuda(), torch.from_numpy(gl).cuda(), None)
    _, v, _ = salgo.online_policy_refinement(graph, max_iter=1, return_info=True)
    keep = torch.nonzero(v == 0).flatten().cpu().numpy()[:E]
    graph = senv.get_graph(torch.from_numpy(ag[keep]).cuda(), torch.from_numpy(gl[keep]).cuda(), None)
    floor = {}
    for mi in (1, 30):
        salgo.online_policy_refinement(graph, max_iter=mi)          # warm-up outside capture
        torch.cuda.synchronize()
        cg = torch.cuda.CUDAGraph()
        with torch.cuda.graph(cg):                                  # as in a rollout: one captured call
            _, v, its = salgo.online_policy_refinement(graph, max_iter=mi, return_info=True)
        cg.replay()
        torch.cuda.synchronize()
        floor[f"max_iter_{mi}"] = {"ms_per_call": _timed(cg.replay, args.floor_calls, args.repeats, clocks),
                                   "iters_max": int(_lib.split_iters(its)[0].max()),
                                   "graphs_value_0": int((v == 0).sum())}
        del cg
    d = float(np.median(floor["max_iter_30"]["ms_per_call"]) - np.median(floor["max_iter_1"]["ms_per_call"]))
    floor.update(graphs=int(len(keep)), pool=pool, note="one captured call: actor forward + planes + refinement of one batch; every graph "
                                "stops at iteration 1", us_per_exited_iteration=d / 29 * 1e3)
    out["early_exit"] = floor
    return _finish(out, clocks)


def _finish(out: dict, clocks: list) -> dict:
    out["clocks"] = clocks
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    out["gpu"] = q.stdout.strip() if q.returncode == 0 else "unknown"
    out["value"] = out["actor_refine"]["value"]
    out["slowdown_vs_actor"] = out["actor"]["value"] / out["actor_refine"]["value"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=3, choices=sorted(CONFIGS))
    ap.add_argument("--envs", type=int, default=None, help="default: the config's envs / its GPU count")
    ap.add_argument("--T", type=int, default=64)
    ap.add_argument("--steps", type=int, default=2, help="refined rollouts per timed window")
    ap.add_argument("--actor-rollouts", type=int, default=100, help="plain-actor rollouts per timed window")
    ap.add_argument("--floor-calls", type=int, default=20, help="refinement calls per timed window (early exit)")
    ap.add_argument("--repeats", type=int, default=3, help="timed windows per row (the spread)")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--weights", type=str, default="both", choices=["both", "pretrained", "xavier"])
    args = ap.parse_args()
    for w in (("pretrained", "xavier") if args.weights == "both" else (args.weights,)):
        print(json.dumps(run(args, w)), flush=True)


if __name__ == "__main__":
    main()
