"""Pieces of tests/test_gpu_resume.py's restore test, and its fresh process: `python resume_worker.py STATE OUT` builds a
new trainer, restores STATE, runs one update on the third rollout and saves the resulting state to OUT."""
import os
import sys

import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

N_ENVS, T = 4, 96        # 384 graphs per rollout: more than a 256-graph minibatch, so the second update samples replay


def setup():
    """A Trainer (no run directory) over a DoubleIntegrator swarm, with a rollout engine of its own."""
    from helpers import product_algo, product_env
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    from gcbfplus_b200.trainer.trainer import Trainer
    env = product_env("DoubleIntegrator", 8, 4.0, 2)
    algo = product_algo(env, seed=0)
    params = {"run_name": "resume", "training_steps": 4, "eval_interval": 1, "eval_epi": 1, "save_interval": 1}
    tr = Trainer(env, product_env("DoubleIntegrator", 8, 4.0, 2), algo, n_env_train=N_ENVS, n_env_test=2, log_dir="",
                 seed=0, params=params, save_log=False)
    tr.engine = RolloutEngine(env, N_ENVS, T=T)
    return tr


def rollout_for(tr, i: int):
    """The i-th training rollout with the trainer's current actor."""
    from gcbfplus_b200.trainer.utils import rollout
    from gcbfplus_b200.utils import jrandom as jr
    return rollout(tr.env, tr.engine, tr.algo.actor_params, jr.split(jr.PRNGKey(100 + i), N_ENVS))


def snapshot(tr, info: dict) -> dict:
    """Everything the next update depends on, as CPU tensors and plain values, plus the last update's info."""
    from gcbfplus_b200.trainer.train_state import state_dict
    torch.cuda.synchronize()
    sd = state_dict(tr, tr.update_steps)
    sd["info"] = {k: float(v) for k, v in info.items()}      # plain floats: the file is read with weights_only
    return sd


def main(state: str, out: str) -> None:
    from gcbfplus_b200.trainer.train_state import load_train_state
    tr = setup()
    load_train_state(tr, state)
    info = tr.algo.update(rollout_for(tr, 2), 2)
    torch.save(snapshot(tr, info), out)


if __name__ == "__main__":
    main(sys.argv[1], sys.argv[2])
