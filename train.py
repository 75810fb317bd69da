"""train.py -- same flags as the reference's train.py:115-151 (+ --cpu which is rejected: the
product path has no CPU fallback; the CPU restatement lives in oracle/ for tests only)."""
import argparse
import datetime
import os

import numpy as np
import yaml

from gcbfplus_b200.algo import make_algo
from gcbfplus_b200.env import make_env
from gcbfplus_b200.trainer.trainer import Trainer


def train(args):
    print(f"> Running train.py {args}")
    if args.cpu:
        raise SystemExit("--cpu: gcbfplus_b200 is the sm_90a CUDA path only (no CPU fallback by design)")
    # before any device, directory or run is set up: the train step implements one GNN layer
    from gcbfplus_b200.algo.train import require_one_layer
    require_one_layer(args.gnn_layers, "training (train.py --gnn-layers)")
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
    log_dir = f"{args.log_dir}/{args.env}/{args.algo}/seed{args.seed}_{start_time}"
    if rank == 0:
        os.makedirs(log_dir, exist_ok=True)
    run_name = f"{args.algo}_{args.env}_{start_time}" if args.name is None else args.name
    train_params = {"run_name": run_name, "training_steps": args.steps, "eval_interval": args.eval_interval,
                    "eval_epi": args.eval_epi, "save_interval": args.save_interval}
    trainer = Trainer(env=env, env_test=env_test, algo=algo, log_dir=log_dir, n_env_train=args.n_env_train,
                      n_env_test=args.n_env_test, seed=args.seed, params=train_params,
                      save_log=not args.debug and rank == 0)
    if not args.debug and rank == 0:
        with open(f"{log_dir}/config.yaml", "w") as f:
            yaml.dump(args, f)
            yaml.dump(algo.config, f)
    trainer.train()


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


def main():
    train(build_parser(FLAGS).parse_args())


if __name__ == "__main__":
    main()
