"""DubinsCar -- gcbfplus/env/dubins_car.py (state [x, y, theta, v], action [omega, acc])."""
import numpy as np
import torch

from .base import MultiAgentEnv


class DubinsCar(MultiAgentEnv):
    AGENT, GOAL, OBS = 0, 1, 2
    ENV_ID = "DubinsCar"
    DIMS = (4, 4, 2, 2)
    PARAMS = {"car_radius": 0.05, "comm_radius": 0.5, "n_rays": 16, "obs_len_range": [0.1, 0.6], "n_obs": 8}

    def _setup_dynamics(self) -> None:
        self.enable_stop = True  # dubins_car.py:54; False (DecShareCBF) turns the stop mask of step() off

    def _thresholds(self) -> dict:
        r = self.radius  # dubins_car.py:398-440
        return dict(unsafe_agent=r * 2, unsafe_obs=r * 1.5, safe_agent=r * 4, safe_obs=r * 2)

    def _reset_extra(self, keys: np.ndarray, agent: np.ndarray, goal: np.ndarray) -> None:
        """dubins_car.py:93-98: random heading from split(key)[0] of the key get_node_goal_rng received;
        goal heading = atan2 towards the goal."""
        from ..utils import jrandom as jr
        theta_key = jr.split(keys, 2)[:, 0]
        agent[:, :, 2] = jr.uniform(theta_key, (agent.shape[1],), -np.pi, np.pi)
        goal[:, :, 2] = np.arctan2(goal[:, :, 1] - agent[:, :, 1], goal[:, :, 0] - agent[:, :, 0])

    def state_lim(self, state=None):
        up = torch.tensor([float("inf"), float("inf"), float("inf"), 0.8])
        return -up, up

    def action_lim(self):
        up = torch.ones(2) * 3.0
        return -up, up

    def control_affine_dyn(self, state: torch.Tensor):
        """dubins_car.py:243-254 (note: omega gain 10 here vs 20 in agent_xdot -- reference quirk)."""
        f = torch.stack([torch.cos(state[..., 2]) * state[..., 3], torch.sin(state[..., 2]) * state[..., 3],
                         torch.zeros_like(state[..., 0]), torch.zeros_like(state[..., 0])], dim=-1)
        g = torch.cat([torch.zeros(2, 2), torch.tensor([[10.0, 0.0], [0.0, 1.0]])], dim=0).to(state.device)
        return f, g.expand(*state.shape[:-1], -1, -1)

    def stop_mask(self, graph) -> torch.Tensor:
        """dubins_car.py:483-487."""
        d = (graph.agent[..., :2] - graph.goal[..., :2]).norm(dim=-1)
        return d < self.radius * 0.5
