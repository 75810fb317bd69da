"""Oracle online policy refinement (TEST INFRASTRUCTURE ONLY): a torch restatement of GCBF.online_policy_refinement
(gcbfplus/algo/gcbf.py:161-201) for ONE graph, on oracle.algo.get_cbf / act, oracle.envs forward_graph / u_ref and
torch.autograd.grad (jax.value_and_grad in the reference), in the dtype of the oracle environment and parameters.

torch's relu differentiates as 1[x > 0] (relu'(0) = 0 and 0 at NaN, like JAX's), clip_action / clip_state pass no
gradient outside their limits, and Python's `nan > 0` is False: an agent at its goal (NaN u_ref) ends the loop after the
mandatory first iteration, as in the reference."""
from __future__ import annotations

import torch

from oracle.algo import get_cbf
from oracle.envs import Graph, OracleEnv
from oracle.nn import net_forward


def refine_value(env: OracleEnv, cbf_p, g: Graph, h: torch.Tensor, a: torch.Tensor, alpha: float) -> torch.Tensor:
    """mean_agents relu(-(cbf(forward_graph(g, a)) - h) / dt - alpha h) (h_dot_cond_val, gcbf.py:182-187)."""
    h_next = get_cbf(cbf_p, env.forward_graph(g, a)).squeeze(-1)
    return torch.relu(-((h_next - h) / env.dt) - alpha * h).mean()


def refine_oracle(env: OracleEnv, cbf_p, actor_p, g: Graph, alpha: float = 1.0, lr: float = 0.1,
                  max_iter: int = 30) -> dict:
    """Returns action [N, nu], iters, the per-iteration loop values (before each update), the per-agent selection
    (v_ref > 0) and its term -(h(g'(u_ref)) - h) / dt - alpha h."""
    with torch.no_grad():
        h = get_cbf(cbf_p, g).squeeze(-1)
        u_ref = env.u_ref(g.agent, g.goal)
        h_ur = get_cbf(cbf_p, env.forward_graph(g, u_ref)).squeeze(-1)
        sel_term = -((h_ur - h) / env.dt) - alpha * h
        sel = torch.relu(sel_term) > 0
        nn_action = 2 * net_forward(actor_p, g, "actor") + u_ref
        a = torch.where(sel[:, None], nn_action, u_ref)
    i, val, values = 0, 1.0, []
    while val > 0 and i < max_iter:
        a_var = a.detach().clone().requires_grad_(True)
        v = refine_value(env, cbf_p, g, h, a_var, alpha)
        (grad,) = torch.autograd.grad(v, a_var)
        a = (a_var - lr * grad).detach()
        val = float(v.detach())
        values.append(val)
        i += 1
    return {"action": a, "iters": i, "values": values, "sel": sel, "sel_term": sel_term, "u_ref": u_ref}
