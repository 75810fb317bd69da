"""test.py -- evaluation CLI with the reference's flags (test.py:239-266): rollouts with a trained
(or --u-ref nominal) controller and safe / finish / success rates (test.py:184-198).
Video rendering is out of scope (SURVEY 2 row 17) -> --no-video is implied; --cbf <agent id> computes the CBF
contour grids the reference hands to its renderer (test.py:125-131, trainer/utils.py:149-168) and saves them as
<path>/cbf_contours/epi<k>_agent<id>.npz (b_xs, b_ys, bb_h per time step).  --nojit-rollout is accepted: the
reference needs it to survive n >= 512 with dense graphs (env/base.py:191-259); the sparse rollout engine has no such limit.
--algo centralized_cbf | dec_share_cbf without --path runs the CBF-QP baseline controllers (test.py:88-103) with
alpha = --alpha and writes to ./logs/<env>/<algo>.
--online-refine (with --path) refines every action of the trained GCBF+ policy against its CBF
(GCBFPlus.online_policy_refinement, gcbf.py:161-201) and prints the refinement's iteration statistics.
--qp-filter (with --path) passes every action of the trained GCBF+ policy through the learned CBF's QP safety filter
(GCBFPlus.safety_filter: the action nearest to 2 pi + u_ref that keeps the CBF condition); with --u-ref as well it
filters u_ref instead (the reference's get_qp_action as a controller).  It prints the QP statistics after the rates.
--all-steps (with --path) evaluates every checkpoint of the run, --paths RUN [RUN ...] the last checkpoint (or --step) of
several runs of one configuration, --paths with --all-steps every checkpoint of each.  All the networks roll out
together (RolloutEngine with n_nets networks: one persistent launch where it applies), each on exactly the episodes
`--path RUN --step S` would give it; one summary line per network, prefixed run=<dir> step=<S>, then the best network
by success rate.  --log appends one row per network (step first, then test_log.csv's columns) to <run>/test_sweep.csv.
--falsify ITERS (with --path) searches for states where the trained CBF's condition fails under the policy
(GCBFPlus.falsify: ITERS normalised gradient-ascent iterations) from every recorded step of the evaluation episodes,
prints one summary line and writes <path>/falsify/step<S>.npz.
--state-noise S [S ...] (one value or state_dim values), --lidar-noise S and --action-noise S [S ...] evaluate the
controller under observation and actuation noise (trainer/rollout.py Perturbation, DESIGN.md 4.11): every agent acts on
x + S z of the agent states and on noisy LiDAR hits, and the applied action is the commanded one plus S z.  The draws
come from --noise-seed (default: --seed) and each episode's index (--offset counts), so an episode gets the same noise
in any batch.  One line reports the sigmas and the realised mean |x_hat - x|; --log writes to test_log_noise.csv, the
sigmas and seed first."""
import argparse
import os

import numpy as np
import yaml

from gcbfplus_b200.algo import make_algo
from gcbfplus_b200.algo.cbf_qp import BASELINES
from gcbfplus_b200.algo.train import QP_MAX_ITER
from gcbfplus_b200.env import make_env
from gcbfplus_b200.trainer.rollout import Perturbation, RolloutEngine
from gcbfplus_b200.trainer.utils import cbf_contours, test_rates


def test(args):
    print(f"> Running test.py {args}")
    if args.cpu:
        raise SystemExit("--cpu: gcbfplus_b200 is the sm_90a CUDA path only (no CPU fallback by design)")
    perturbation = noise_perturbation(args)
    check_falsify_flags(args)
    if check_sweep_flags(args):
        test_sweep(args)
        return
    check_qp_filter_flags(args)
    check_refine_flags(args)
    np.random.seed(args.seed)
    config = None
    trained = args.path is not None and (not args.u_ref or args.qp_filter)
    if trained:
        with open(os.path.join(args.path, "config.yaml"), "r") as f:
            config = yaml.load(f, Loader=yaml.UnsafeLoader)
    num_agents = config.num_agents if args.num_agents is None else args.num_agents
    env = make_env(env_id=config.env if args.env is None else args.env, num_agents=num_agents, num_obs=args.obs,
                   area_size=args.area_size, max_step=args.max_step, max_travel=args.max_travel)
    if perturbation is not None:
        try:
            perturbation.sigmas(env)
        except ValueError as e:
            raise SystemExit(f"noise flags: {e}")
    policy = "u_ref"
    algo = None
    baseline = args.algo in BASELINES and args.path is None and not args.u_ref
    if baseline:
        if args.cbf is not None:
            raise SystemExit(f"--cbf: the CBF contours are not available for the {args.algo} baseline (the reference's "
                             "contour path only works with a trained GCBF+ CBF)")
        assert args.env is not None, "--env required for a baseline"
        algo = make_algo(algo=args.algo, env=env, node_dim=env.node_dim, edge_dim=env.edge_dim,
                         state_dim=env.state_dim, action_dim=env.action_dim, n_agents=env.num_agents, alpha=args.alpha)
        policy = algo
        path = os.path.join(f"./logs/{args.env}/{args.algo}")
        os.makedirs(path, exist_ok=True)
    elif trained or not args.u_ref:
        assert args.path is not None, "--path or --u-ref required"
        model_path = os.path.join(args.path, "models")
        step = max(int(m) for m in os.listdir(model_path) if m.isdigit()) if args.step is None else args.step
        print("step: ", step)
        algo = make_algo(
            algo=config.algo, env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
            action_dim=env.action_dim, n_agents=env.num_agents, gnn_layers=config.gnn_layers,
            batch_size=config.batch_size, buffer_size=config.buffer_size, horizon=config.horizon,
            lr_actor=config.lr_actor, lr_cbf=config.lr_cbf, alpha=config.alpha, eps=0.02, inner_epoch=8,
            loss_action_coef=config.loss_action_coef, loss_unsafe_coef=config.loss_unsafe_coef,
            loss_safe_coef=config.loss_safe_coef, loss_h_dot_coef=config.loss_h_dot_coef, max_grad_norm=2.0,
            seed=config.seed)
        algo.load(model_path, step)
        if args.qp_filter:
            policy = "u_ref_qp" if args.u_ref else "actor_qp"
        else:
            policy = "actor_refine" if args.online_refine else "actor"
        path = args.path
    else:
        assert args.env is not None
        path = os.path.join(f"./logs/{args.env}/nominal")
        os.makedirs(path, exist_ok=True)
    n_epi = args.epi - args.offset
    eng = RolloutEngine(env, n_epi, T=env.max_episode_steps, policy=policy, perturbation=perturbation)
    if algo is not None and not baseline:
        eng.set_params(algo.actor_params)
        if args.online_refine or args.qp_filter:
            eng.set_cbf_params(algo.cbf_params, alpha=algo.alpha)
    # test.py:117-119,158: test_keys = split(PRNGKey(seed), 1000)[:epi][offset:]; episode i resets with
    # split(test_keys[i])[0].  All episodes run as one batch here.
    from gcbfplus_b200.utils import jrandom as jr
    test_keys = jr.split(jr.PRNGKey(args.seed), 1_000)[: args.epi][args.offset:]
    g0 = env.reset(jr.split(test_keys, 2)[:, 0])
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    ro = eng.result()
    summary = summarize(env, ro)
    rates, rewards, costs = summary["rates"], summary["rewards"], summary["costs"]
    for i in range(n_epi):
        print(f"epi: {i}, reward: {rewards[i]:.3f}, cost: {costs[i]:.3f}, safe rate: {rates[i, 0] * 100:.3f}%,"
              f"finish rate: {rates[i, 1] * 100:.3f}%, success rate: {rates[i, 2] * 100:.3f}%")
    print(summary["line"])
    if perturbation is not None:
        sx, sl, su = perturbation.sigmas(env)
        err = float((eng.obs_agent - eng.agent[:-1]).abs().mean())
        print(f"noise: state sigma {sx}, LiDAR sigma {sl}, action sigma {su}, seed {perturbation.seed}; "
              f"realised mean |x_hat - x| {err:.6f}")
    if baseline or args.qp_filter:
        st = eng.qp_stats()
        print(f"QP iterations: median {st['iters_median']:.0f}, max {st['iters_max']}, "
              f"capped {st['capped']} of {st['solves']} solves")
        if args.qp_filter:
            print(f"QP filter: mean |u - u_nom| {st['mean_correction']:.4f}, CBF condition relaxed (r > 0) in "
                  f"{st['relaxed_frac'] * 100:.3f}% of agent-steps")
        if st["capped"]:
            cap = QP_MAX_ITER if args.qp_filter else algo.max_iter
            print(f"WARNING: {st['capped']} QP solve(s) hit the iteration cap ({cap}); their actions are the "
                  "capped iterates, not the exact QP minimisers")
    if args.online_refine:
        st = eng.refine_stats()
        print(f"refinement iterations: median {st['iters_median']:.0f}, max {st['iters_max']}, "
              f"capped {st['capped']} of {st['graph_steps']} graph-steps")
        if st["capped"]:
            print(f"WARNING: {st['capped']} graph-step(s) hit the refinement cap ({eng.refine_max_iter} iterations) "
                  "with the CBF condition still violated; their actions are the capped iterates")
    if args.log and perturbation is not None:
        sx, sl, su = perturbation.sigmas(env)
        with open(os.path.join(path, "test_log_noise.csv"), "a") as f:
            f.write(f"{' '.join(map(str, sx))},{sl},{' '.join(map(str, su))},{perturbation.seed},"
                    + log_row(env, args, summary) + "\n")
    elif args.log:
        with open(os.path.join(path, "test_log.csv"), "a") as f:
            f.write(log_row(env, args, summary) + "\n")
    if getattr(args, "falsify", None) is not None:
        run_falsify(args, env, algo, eng, g0, path, step)
    if args.cbf is not None:
        assert algo is not None, "--cbf needs a trained CBF (--path)"
        out_dir = os.path.join(path, "cbf_contours")
        os.makedirs(out_dir, exist_ok=True)
        for i in range(n_epi):
            b_x, b_y, bb_h = cbf_contours(algo, env, ro, i, args.cbf)
            f_out = os.path.join(out_dir, f"epi{i + args.offset:02}_agent{args.cbf}.npz")
            np.savez_compressed(f_out, b_xs=b_x, b_ys=b_y, bb_h=bb_h, agent_id=args.cbf)
            print(f"cbf contour grid: {f_out} {bb_h.shape}")
    if not args.no_video:
        print("video rendering is out of scope of the CUDA hot path (SURVEY.md section 2, row 17); skipped")


def summarize(env, ro) -> dict:
    """Per-episode rates / rewards / costs of a rollout and the means test.py prints and logs (test.py:184-198)."""
    rates, is_unsafe, is_finish = test_rates(env, ro)
    rewards = ro.rewards.sum(dim=1).cpu().numpy()
    costs = ro.costs.sum(dim=1).cpu().numpy()
    succ = (1 - is_unsafe) * is_finish
    st = dict(rates=rates, rewards=rewards, costs=costs, safe=(1 - is_unsafe).mean(), safe_std=(1 - is_unsafe).std(),
              finish=is_finish.mean(), finish_std=is_finish.std(), success=succ.mean(), success_std=succ.std())
    st["line"] = (f"reward: {np.mean(rewards):.3f}, min/max reward: {np.min(rewards):.3f}/{np.max(rewards):.3f}, "
                  f"cost: {np.mean(costs):.3f}, min/max cost: {np.min(costs):.3f}/{np.max(costs):.3f}, "
                  f"safe_rate: {st['safe'] * 100:.3f}%, finish_rate: {st['finish'] * 100:.3f}%, "
                  f"success_rate: {st['success'] * 100:.3f}%")
    return st


def log_row(env, args, st) -> str:
    """One test_log.csv row: the setting, then the safe / finish / success means and spreads in percent."""
    return (f"{env.num_agents},{args.epi},{env.max_episode_steps},{env.area_size},{env.params['n_obs']},"
            f"{st['safe'] * 100:.3f},{st['safe_std'] * 100:.3f},{st['finish'] * 100:.3f},{st['finish_std'] * 100:.3f},"
            f"{st['success'] * 100:.3f},{st['success_std'] * 100:.3f}")


#: config.yaml keys every run of one --paths sweep must share: they fix the environment and the network shape
SWEEP_KEYS = ("env", "num_agents", "gnn_layers", "n_rays")


def check_sweep_flags(args) -> bool:
    """--all-steps / --paths evaluate the trained actors of one or more runs together.  Returns whether the invocation
    is such a sweep; refuses the combinations it does not implement.  (A namespace parsed from FLAGS alone has neither
    flag: not a sweep.)"""
    args.paths, args.all_steps = getattr(args, "paths", None), getattr(args, "all_steps", False)
    if args.paths is None and not args.all_steps:
        return False
    if args.paths is not None and args.path is not None:
        raise SystemExit("--paths and --path are mutually exclusive: give the runs with one of them")
    if args.paths is None and args.path is None:
        raise SystemExit("--all-steps needs a trained GCBF+ run (--path or --paths)")
    what = "--all-steps" if args.paths is None else "--paths"
    if args.all_steps and args.step is not None:
        raise SystemExit("--all-steps evaluates every checkpoint; it cannot be combined with --step")
    for flag, given in (("--u-ref", args.u_ref), ("--online-refine", args.online_refine),
                        ("--qp-filter", args.qp_filter), ("--cbf", args.cbf is not None)):
        if given:
            raise SystemExit(f"{what} evaluates the trained actors of many checkpoints; it cannot be combined with {flag}")
    if args.algo in BASELINES:
        raise SystemExit(f"{what} evaluates trained GCBF+ actors; it cannot be combined with the {args.algo} baseline "
                         "(--algo)")
    return True


def checkpoint_steps(run: str) -> list:
    """The numeric checkpoint directories under <run>/models, ascending."""
    model_path = os.path.join(run, "models")
    steps = sorted(int(m) for m in os.listdir(model_path) if m.isdigit()) if os.path.isdir(model_path) else []
    if not steps:
        raise SystemExit(f"{run}: no checkpoints under {model_path}")
    return steps


def read_config(run: str):
    with open(os.path.join(run, "config.yaml"), "r") as f:
        return yaml.load(f, Loader=yaml.UnsafeLoader)


def check_sweep_configs(runs: list, configs: list) -> None:
    """Every run of a sweep shares SWEEP_KEYS with the first one; the refusal names the key that differs."""
    for run, cfg in zip(runs[1:], configs[1:]):
        for key in SWEEP_KEYS:
            a, b = getattr(configs[0], key, None), getattr(cfg, key, None)
            if a != b:
                raise SystemExit(f"--paths: {run} has {key} = {b!r} but {runs[0]} has {key} = {a!r}; the runs of one "
                                 "sweep must share " + ", ".join(SWEEP_KEYS))


def sweep_networks(args, runs: list) -> list:
    """(run, step) of every network of the sweep: all checkpoints with --all-steps, else --step or the last one."""
    nets = []
    for run in runs:
        steps = checkpoint_steps(run)
        for step in steps if args.all_steps else [steps[-1] if args.step is None else args.step]:
            nets.append((run, step))
    return nets


def test_sweep(args):
    """--all-steps / --paths: every network on the episodes a solo `--path RUN --step S` run gives it, in one rollout."""
    np.random.seed(args.seed)
    runs = args.paths if args.paths is not None else [args.path]
    configs = [read_config(r) for r in runs]
    check_sweep_configs(runs, configs)
    nets = sweep_networks(args, runs)
    config = configs[0]
    num_agents = config.num_agents if args.num_agents is None else args.num_agents
    env = make_env(env_id=config.env if args.env is None else args.env, num_agents=num_agents, num_obs=args.obs,
                   area_size=args.area_size, max_step=args.max_step, max_travel=args.max_travel)
    params, algos = [], {}
    for run, step in nets:
        if run not in algos:
            cfg = configs[runs.index(run)]
            algos[run] = make_algo(
                algo=cfg.algo, env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                action_dim=env.action_dim, n_agents=env.num_agents, gnn_layers=cfg.gnn_layers,
                batch_size=cfg.batch_size, buffer_size=cfg.buffer_size, horizon=cfg.horizon, lr_actor=cfg.lr_actor,
                lr_cbf=cfg.lr_cbf, alpha=cfg.alpha, eps=0.02, inner_epoch=8, loss_action_coef=cfg.loss_action_coef,
                loss_unsafe_coef=cfg.loss_unsafe_coef, loss_safe_coef=cfg.loss_safe_coef,
                loss_h_dot_coef=cfg.loss_h_dot_coef, max_grad_norm=2.0, seed=cfg.seed)
        algos[run].load(os.path.join(run, "models"), step)
        params.append(algos[run].actor_params.clone())
    K, n_epi = len(nets), args.epi - args.offset
    print(f"networks: {K}, episodes per network: {n_epi}")
    # network k runs environments [k n_epi, (k + 1) n_epi): the same initial states for every network (test.py:117-119)
    eng = RolloutEngine(env, K * n_epi, T=env.max_episode_steps, policy="actor", n_nets=K)
    eng.set_params(params)
    from gcbfplus_b200.utils import jrandom as jr
    test_keys = jr.split(jr.PRNGKey(args.seed), 1_000)[: args.epi][args.offset:]
    g0 = env.reset(jr.split(test_keys, 2)[:, 0])
    obstacle = g0.obstacle.repeat(K) if hasattr(g0.obstacle, "repeat") else g0.obstacle
    eng.set_initial(g0.agent.repeat(K, 1, 1), g0.goal.repeat(K, 1, 1), obstacle)
    eng.run()
    best = None
    for k, (run, step) in enumerate(nets):
        st = summarize(env, eng.net_result(k))
        print(f"run={run} step={step} " + st["line"])
        if best is None or st["success"] > best[2]:
            best = (run, step, st["success"])
        if args.log:
            with open(os.path.join(run, "test_sweep.csv"), "a") as f:
                f.write(f"{step}," + log_row(env, args, st) + "\n")
    print(f"best: run={best[0]} step={best[1]} success_rate: {best[2] * 100:.3f}%")
    if not args.no_video:
        print("video rendering is out of scope of the CUDA hot path (SURVEY.md section 2, row 17); skipped")


def check_falsify_flags(args) -> None:
    """--falsify ITERS searches a trained GCBF+ run's CBF (--path) for counterexamples from the states its actor visits:
    it excludes every other controller and the sweeps."""
    if getattr(args, "falsify", None) is None:
        return
    if args.falsify < 1:
        raise SystemExit(f"--falsify takes the number of search iterations (>= 1), got {args.falsify}")
    for flag, given in (("--u-ref", args.u_ref), ("--online-refine", args.online_refine),
                        ("--qp-filter", args.qp_filter), ("--paths", getattr(args, "paths", None) is not None),
                        ("--all-steps", getattr(args, "all_steps", False))):
        if given:
            raise SystemExit(f"--falsify searches the CBF of one trained GCBF+ actor; it cannot be combined with {flag}")
    if args.algo in BASELINES:
        raise SystemExit(f"--falsify searches a trained GCBF+ CBF; it cannot be combined with the {args.algo} baseline")
    if args.path is None:
        raise SystemExit("--falsify needs a trained GCBF+ run (--path)")


def run_falsify(args, env, algo, eng, g0, path: str, step: int) -> None:
    """--falsify: the search from every recorded state of the episodes (each with its own goals and obstacles), one
    summary line, and the per-graph results in <path>/falsify/step<S>.npz (graph g = t * n_epi + e)."""
    import torch
    states = eng.agent                                          # [T + 1, E, N, sd]
    T1, E = states.shape[0], states.shape[1]
    agent = states.reshape(T1 * E, *states.shape[2:]).contiguous()
    goal = g0.goal.repeat(T1, 1, 1).contiguous()
    obstacle = g0.obstacle.repeat(T1) if g0.obstacle is not None else None
    r = algo.falsify(agent, goal, obstacle, args.falsify)
    torch.cuda.synchronize()
    n = agent.shape[0]
    n_agents = n * env.num_agents
    viol0 = float((r["J0"] > 0).float().mean()) * 100
    viol = float((r["J"] > 0).float().mean()) * 100
    print(f"falsify: {n} graphs searched ({args.falsify} iterations), CBF condition violated in {viol0:.3f}% at the "
          f"start and {viol:.3f}% after the search, largest term {float(r['J'].max()):.4f}, false-safe "
          f"{r['false_safe0'] / n_agents * 100:.3f}% at the start and {r['false_safe'] / n_agents * 100:.3f}% at the "
          f"found states")
    out_dir = os.path.join(path, "falsify")
    os.makedirs(out_dir, exist_ok=True)
    f_out = os.path.join(out_dir, f"step{step}.npz")
    np.savez_compressed(f_out, **{k: v.cpu().numpy() for k, v in r.items() if torch.is_tensor(v)},
                        goal=goal.cpu().numpy(), false_safe0=r["false_safe0"], false_safe=r["false_safe"],
                        n_iter=args.falsify)
    print(f"falsify results: {f_out}")


NOISE_FLAGS = (("--state-noise", "state_noise"), ("--lidar-noise", "lidar_noise"), ("--action-noise", "action_noise"))


def noise_perturbation(args):
    """The Perturbation of --state-noise / --lidar-noise / --action-noise (None without them): checked before any device
    work.  Noisy evaluation runs one engine on the step-by-step path, so the sweeps and --falsify (which searches from
    the noiseless states) are refused, naming the flag.  (A namespace parsed from FLAGS alone has none of the flags.)"""
    given = [flag for flag, key in NOISE_FLAGS if getattr(args, key, None) is not None]
    seed = getattr(args, "noise_seed", None)
    if not given:
        if seed is not None:
            raise SystemExit("--noise-seed seeds the noise of --state-noise / --lidar-noise / --action-noise; give one "
                             "of them")
        return None
    for flag, on in (("--paths", getattr(args, "paths", None) is not None),
                     ("--all-steps", getattr(args, "all_steps", False)),
                     ("--falsify", getattr(args, "falsify", None) is not None)):
        if on:
            raise SystemExit(f"{given[0]} evaluates one controller under noise; it cannot be combined with {flag}")
    try:
        return Perturbation(args.state_noise if args.state_noise is not None else 0.0,
                            args.lidar_noise if args.lidar_noise is not None else 0.0,
                            args.action_noise if args.action_noise is not None else 0.0,
                            seed=args.seed if seed is None else seed, env_offset=args.offset)
    except ValueError as e:
        raise SystemExit(f"noise flags: {e}")


def check_refine_flags(args) -> None:
    """--online-refine refines a trained GCBF+ policy: it needs --path and excludes --u-ref and the baselines."""
    if not args.online_refine:
        return
    if args.u_ref:
        raise SystemExit("--online-refine refines a trained GCBF+ policy; it cannot be combined with --u-ref")
    if args.path is None:
        if args.algo in BASELINES:
            raise SystemExit(f"--online-refine refines a trained GCBF+ policy; it cannot be combined with the "
                             f"{args.algo} baseline")
        raise SystemExit("--online-refine needs a trained GCBF+ run (--path)")


def check_qp_filter_flags(args) -> None:
    """--qp-filter filters through a trained GCBF+ CBF: it needs --path and excludes --online-refine and the
    baselines (--u-ref selects u_ref as the nominal action)."""
    if not args.qp_filter:
        return
    if args.online_refine:
        raise SystemExit("--qp-filter and --online-refine both correct the policy's action; give one of them")
    if args.algo in BASELINES:
        raise SystemExit(f"--qp-filter filters through a trained GCBF+ CBF; it cannot be combined with the {args.algo} "
                         "baseline")
    if args.path is None:
        raise SystemExit("--qp-filter needs a trained GCBF+ run (--path)")


# the reference's command line (test.py:239-266), table-driven like train.py
FLAGS = [
    (("-n", "--num-agents"), int, None), (("--obs",), int, 0), (("--area-size",), float, "required"),
    (("--max-step",), int, None), (("--path",), str, None), (("--n-rays",), int, 32), (("--alpha",), float, 1.0),
    (("--max-travel",), float, None), (("--cbf",), int, None), (("--seed",), int, 1234), (("--debug",), "flag", False),
    (("--cpu",), "flag", False), (("--u-ref",), "flag", False), (("--env",), str, None), (("--algo",), str, None),
    (("--step",), int, None), (("--epi",), int, 5), (("--offset",), int, 0), (("--no-video",), "flag", False),
    (("--nojit-rollout",), "flag", False), (("--log",), "flag", False), (("--dpi",), int, 100),
    (("--online-refine",), "flag", False), (("--qp-filter",), "flag", False), (("--falsify",), int, None),
]


def build_test_parser():
    """FLAGS plus the sweep flags (--paths takes several runs) and the noise flags (the sigmas take one or more values)."""
    from train import build_parser
    parser = build_parser(FLAGS)
    parser.add_argument("--paths", type=str, nargs="+", default=None)
    parser.add_argument("--all-steps", action="store_true", default=False)
    parser.add_argument("--state-noise", type=float, nargs="+", default=None)
    parser.add_argument("--lidar-noise", type=float, default=None)
    parser.add_argument("--action-noise", type=float, nargs="+", default=None)
    parser.add_argument("--noise-seed", type=int, default=None)
    return parser


def main():
    test(build_test_parser().parse_args())


if __name__ == "__main__":
    main()
