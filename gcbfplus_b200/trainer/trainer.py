"""Trainer -- gcbfplus/trainer/trainer.py:18-143 on the CUDA rollout engine + CUDA train step.
wandb logging is optional (offline / absent -> metrics are printed and kept in `self.history`)."""
from __future__ import annotations

import os
from time import time
from typing import Optional

import numpy as np

from .. import dist as gdist
from ..algo.train import require_one_layer
from ..utils import jrandom as jr
from .rollout import RolloutEngine
from .train_state import load_train_state, save_run_state
from .utils import eval_metrics, rollout


class Trainer:

    def __init__(self, env, env_test, algo, n_env_train: int, n_env_test: int, log_dir: str, seed: int, params: dict,
                 save_log: bool = True, state_dir: Optional[str] = None, resume_from: Optional[str] = None):
        """state_dir: every rank saves its training state there with every model save (trainer/train_state.py).
        resume_from: this rank's saved state file; train() restores it after building its rollout engines and
        continues from its step."""
        # reject a network the train step cannot train before any directory, checkpoint or rollout is made
        require_one_layer(algo.cbf_params.n_layers, "Trainer")
        self.env = env
        self.env_test = env_test
        self.algo = algo
        self.n_env_train = n_env_train
        self.n_env_test = n_env_test
        self.log_dir = log_dir
        self.seed = seed
        if Trainer._check_params(params):
            self.params = params
        if save_log:
            os.makedirs(log_dir, exist_ok=True)
            self.model_dir = os.path.join(log_dir, "models")
            os.makedirs(self.model_dir, exist_ok=True)
        self.wandb = None
        if os.environ.get("WANDB_MODE", "disabled") != "disabled":
            try:
                import wandb
                wandb.init(name=params["run_name"], project="gcbf-b200", dir=self.log_dir)
                self.wandb = wandb
            except Exception as e:  # pragma: no cover
                print(f"wandb unavailable ({e}); logging to stdout only")
        self.save_log = save_log
        self.steps = params["training_steps"]
        self.eval_interval = params["eval_interval"]
        self.eval_epi = params["eval_epi"]
        self.save_interval = params["save_interval"]
        self.update_steps = 0
        self.key = jr.PRNGKey(seed)                                   # trainer.py:62 key stream
        self.history = []
        self.start_step = 0
        self.state_dir = state_dir
        self.resume_from = resume_from

    @staticmethod
    def _check_params(params: dict) -> bool:
        """trainer/trainer.py:64-74."""
        assert "run_name" in params, "run_name not found in params"
        assert "training_steps" in params, "training_steps not found in params"
        assert "eval_interval" in params, "eval_interval not found in params"
        assert params["eval_interval"] > 0, "eval_interval must be positive"
        assert "eval_epi" in params, "eval_epi not found in params"
        assert params["eval_epi"] >= 1, "eval_epi must be greater than or equal to 1"
        assert "save_interval" in params, "save_interval not found in params"
        assert params["save_interval"] > 0, "save_interval must be positive"
        return True

    def _log(self, info: dict) -> None:
        self.history.append(dict(info, update_steps=self.update_steps))
        if self.wandb is not None:
            self.wandb.log(info, step=self.update_steps)

    def train(self):
        """trainer/trainer.py:76-143."""
        start_time = time()
        # one process per GPU (torchrun): the training environments are sharded, every rank evaluates the (small)
        # test set, rank 0 logs and saves; gradients meet in algo.update's single all-reduce per optimizer step
        world = gdist.world_size()
        rank = gdist.dist.get_rank() if world > 1 else 0
        assert self.n_env_train % world == 0, "n_env_train must be divisible by the number of GPUs"
        lo, hi = gdist.shard_bounds(self.n_env_train, rank, world)
        train_engine = RolloutEngine(self.env, hi - lo)
        test_engine = RolloutEngine(self.env_test, self.n_env_test)
        test_keys = jr.split(jr.PRNGKey(self.seed), 1_000)[:self.n_env_test]       # trainer.py:99-100
        if self.resume_from is not None:
            # after the engines: they were built with the edge capacity the run started with, which the state may grow
            load_train_state(self, self.resume_from)
        for step in range(self.start_step, self.steps + 1):
            if step % self.eval_interval == 0:
                ro = rollout(self.env_test, test_engine, self.algo.actor_params, test_keys)
                info = eval_metrics(self.env_test, ro)
                eval_info = {k: v for k, v in info.items() if k.startswith("eval/")}
                eval_info["step"] = step
                self._log(eval_info)
                if rank == 0:
                    print(f"step: {step:3}, time: {time() - start_time:5.0f}s, reward: {info['eval/reward']:9.4f}, "
                          f"min/max reward: {info['reward_min']:7.2f}/{info['reward_max']:7.2f}, "
                          f"cost: {info['eval/cost']:8.4f}, unsafe_frac: {info['eval/unsafe_frac']:6.2f}, "
                          f"finish: {info['eval/finish']:6.2f}")
                if self.save_log and rank == 0 and step % self.save_interval == 0:
                    self.algo.save(os.path.join(self.model_dir), step)
                if self.state_dir is not None and step % self.save_interval == 0:
                    save_run_state(self, self.state_dir, step)
            key_x0, self.key = jr.split(self.key)                     # trainer.py:134-136
            ro = rollout(self.env, train_engine, self.algo.actor_params, jr.split(key_x0, self.n_env_train)[lo:hi])
            update_info = self.algo.update(ro, step)
            self._log(update_info)
            self.update_steps += 1
