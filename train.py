"""train.py -- same flags as the reference's train.py:115-151 (+ --cpu which is rejected: the
product path has no CPU fallback; the CPU restatement lives in oracle/ for tests only), and resume:
--save-state writes the full training state with every model save, --resume RUN_DIR continues that run bit for bit
(DESIGN §4.8)."""
import argparse
import datetime
import os

import numpy as np
import yaml

from gcbfplus_b200.algo import make_algo
from gcbfplus_b200.env import make_env
from gcbfplus_b200.trainer import train_state
from gcbfplus_b200.trainer.trainer import Trainer

# flags of one invocation rather than of the run: config.yaml does not record them
INVOCATION_FLAGS = ("resume", "save_state")


def train(args):
    print(f"> Running train.py {args}")
    if args.cpu:
        raise SystemExit("--cpu: gcbfplus_b200 is the sm_90a CUDA path only (no CPU fallback by design)")
    # before any device, directory or run is set up: the train step implements one GNN layer
    from gcbfplus_b200.algo.train import require_one_layer
    require_one_layer(args.gnn_layers, "training (train.py --gnn-layers)")
    if args.save_state and args.debug:
        raise SystemExit("--save-state: --debug writes no run directory (no config.yaml, no models) to resume from")
    state_file = None
    if args.resume is not None:
        state_file = check_resume(args)
    os.environ.setdefault("WANDB_MODE", "offline")
    # one process per GPU under torchrun (python -m torch.distributed.run --nproc-per-node N train.py ...):
    # environments are sharded over the ranks, gradients all-reduced once per optimizer step (SURVEY 8e)
    import torch
    from gcbfplus_b200 import dist as gdist
    rank, local_rank, world = gdist.init_from_env()
    # replay sampling draws from NumPy's global RNG (trainer/buffer.py:82-87, seeded at train.py:22 in the reference):
    # rank 0 keeps the reference's stream, the other ranks sample their own replay with an offset seed
    np.random.seed(args.seed + rank)
    device = torch.device("cuda", local_rank)
    if args.debug or rank != 0:
        os.environ["WANDB_MODE"] = "disabled"
    env = make_env(env_id=args.env, num_agents=args.num_agents, num_obs=args.obs, n_rays=args.n_rays,
                   area_size=args.area_size, device=device)
    env_test = make_env(env_id=args.env, num_agents=args.num_agents, num_obs=args.obs, n_rays=args.n_rays,
                        area_size=args.area_size, device=device)
    algo = make_algo(
        algo=args.algo, env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
        action_dim=env.action_dim, n_agents=env.num_agents, gnn_layers=args.gnn_layers, batch_size=256,
        buffer_size=args.buffer_size, horizon=args.horizon, lr_actor=args.lr_actor, lr_cbf=args.lr_cbf,
        alpha=args.alpha, eps=0.02, inner_epoch=8, loss_action_coef=args.loss_action_coef,
        loss_unsafe_coef=args.loss_unsafe_coef, loss_safe_coef=args.loss_safe_coef,
        loss_h_dot_coef=args.loss_h_dot_coef, max_grad_norm=2.0, seed=args.seed)
    start_time = datetime.datetime.now().strftime("%Y%m%d%H%M%S")
    log_dir = args.resume if args.resume is not None else \
        f"{args.log_dir}/{args.env}/{args.algo}/seed{args.seed}_{start_time}"
    if world > 1 and args.save_state:
        # every rank writes its training state into the run directory: take rank 0's name (its clock, its start time)
        sync = [log_dir]
        gdist.dist.broadcast_object_list(sync, src=0)
        log_dir = sync[0]
    if rank == 0:
        os.makedirs(log_dir, exist_ok=True)
    run_name = f"{args.algo}_{args.env}_{start_time}" if args.name is None else args.name
    train_params = {"run_name": run_name, "training_steps": args.steps, "eval_interval": args.eval_interval,
                    "eval_epi": args.eval_epi, "save_interval": args.save_interval}
    trainer = Trainer(env=env, env_test=env_test, algo=algo, log_dir=log_dir, n_env_train=args.n_env_train,
                      n_env_test=args.n_env_test, seed=args.seed, params=train_params,
                      save_log=not args.debug and rank == 0,
                      state_dir=os.path.join(log_dir, train_state.STATE_DIR) if args.save_state else None,
                      resume_from=state_file)
    if not args.debug and rank == 0 and args.resume is None:
        write_config(log_dir, args, algo.config)
    trainer.train()


def write_config(log_dir: str, args, algo_config: dict) -> None:
    """<run>/config.yaml: the run's flags (not the per-invocation --resume / --save-state), then the algorithm's
    config; test.py and --resume read it back as one namespace."""
    run_args = argparse.Namespace(**{k: v for k, v in vars(args).items() if k not in INVOCATION_FLAGS})
    with open(f"{log_dir}/config.yaml", "w") as f:
        yaml.dump(run_args, f)
        yaml.dump(algo_config, f)


def check_resume(args) -> str:
    """--resume RUN_DIR: this rank's state file of the run's latest complete training state.  Reads small files only,
    so a run that cannot resume stops before any device work or write."""
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    state_dir = os.path.join(args.resume, train_state.STATE_DIR)
    try:
        latest = train_state.check_resume(state_dir, world)
    except ValueError as e:
        raise SystemExit(f"--resume {args.resume}: {e}") from None
    if args.steps < latest["step"]:
        raise SystemExit(f"--resume {args.resume}: --steps {args.steps} is below the saved step {latest['step']}")
    return train_state.state_file(state_dir, latest["step"], rank)


# (flags, type or "flag", default) -- the reference's command line (train.py:115-151), table-driven
FLAGS = [
    (("-n", "--num-agents"), int, 8), (("--algo",), str, "gcbf+"), (("--env",), str, "SimpleCar"), (("--seed",), int, 0),
    (("--steps",), int, 1000), (("--name",), str, None), (("--debug",), "flag", False), (("--obs",), int, None),
    (("--n-rays",), int, 32), (("--area-size",), float, "required"),
    # GCBF / GCBF+ hyper-parameters
    (("--gnn-layers",), int, 1), (("--alpha",), float, 1.0), (("--horizon",), int, 32), (("--lr-actor",), float, 3e-5),
    (("--lr-cbf",), float, 3e-5), (("--loss-action-coef",), float, 1e-4), (("--loss-unsafe-coef",), float, 1.0),
    (("--loss-safe-coef",), float, 1.0), (("--loss-h-dot-coef",), float, 0.01), (("--buffer-size",), int, 512),
    # run control
    (("--n-env-train",), int, 16), (("--n-env-test",), int, 32), (("--log-dir",), str, "./logs"),
    (("--eval-interval",), int, 1), (("--eval-epi",), int, 1), (("--save-interval",), int, 10), (("--cpu",), "flag", False),
    # resume: --save-state writes the training state with every model save, --resume RUN_DIR continues that run
    (("--save-state",), "flag", False), (("--resume",), str, None),
]


def build_parser(flags) -> argparse.ArgumentParser:
    parser = argparse.ArgumentParser()
    for names, kind, default in flags:
        if kind == "flag":
            parser.add_argument(*names, action="store_true", default=default)
        elif default == "required":
            parser.add_argument(*names, type=kind, required=True)
        else:
            parser.add_argument(*names, type=kind, default=default)
    return parser


def parse_args(argv=None) -> argparse.Namespace:
    """The command line.  With --resume RUN_DIR every flag comes from the run's config.yaml (read as test.py reads it);
    only --steps may be given, to extend the run.  The resumed run keeps saving its training state."""
    pre = argparse.ArgumentParser(add_help=False)
    pre.add_argument("--resume", type=str, default=None)
    run_dir = pre.parse_known_args(argv)[0].resume
    if run_dir is None:
        return build_parser(FLAGS).parse_args(argv)
    given = argparse.ArgumentParser(argument_default=argparse.SUPPRESS)
    for names, kind, _ in FLAGS:
        given.add_argument(*names, **({"action": "store_true"} if kind == "flag" else {"type": kind}))
    given = vars(given.parse_args(argv))
    extra = sorted(set(given) - {"resume", "steps"})
    if extra:
        raise SystemExit(f"--resume takes every flag from {run_dir}/config.yaml; only --steps may be given, got "
                         + ", ".join("--" + k.replace("_", "-") for k in extra))
    try:
        with open(os.path.join(run_dir, "config.yaml"), "r") as f:
            args = yaml.load(f, Loader=yaml.UnsafeLoader)
    except OSError as e:
        raise SystemExit(f"--resume {run_dir}: cannot read the run's config.yaml ({e})") from None
    args.resume, args.save_state = run_dir, True
    args.steps = given.get("steps", args.steps)
    return args


def main():
    train(parse_args())


if __name__ == "__main__":
    main()
