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
by success rate.  --log appends one row per network (step first, then test_log.csv's columns) to <run>/test_sweep.csv."""
import argparse
import os

import numpy as np
import yaml

from gcbfplus_b200.algo import make_algo
from gcbfplus_b200.algo.cbf_qp import BASELINES
from gcbfplus_b200.algo.train import QP_MAX_ITER
from gcbfplus_b200.env import make_env
from gcbfplus_b200.trainer.rollout import RolloutEngine
from gcbfplus_b200.trainer.utils import cbf_contours, test_rates


def test(args):
    print(f"> Running test.py {args}")
    if args.cpu:
        raise SystemExit("--cpu: gcbfplus_b200 is the sm_90a CUDA path only (no CPU fallback by design)")
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
    eng = RolloutEngine(env, n_epi, T=env.max_episode_steps, policy=policy)
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
    if args.log:
        with open(os.path.join(path, "test_log.csv"), "a") as f:
            f.write(log_row(env, args, summary) + "\n")
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
    (("--online-refine",), "flag", False), (("--qp-filter",), "flag", False),
]


def build_test_parser():
    """FLAGS plus the sweep flags (--paths takes several runs)."""
    from train import build_parser
    parser = build_parser(FLAGS)
    parser.add_argument("--paths", type=str, nargs="+", default=None)
    parser.add_argument("--all-steps", action="store_true", default=False)
    return parser


def main():
    test(build_test_parser().parse_args())


if __name__ == "__main__":
    main()
