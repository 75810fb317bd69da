"""GPU parity: GNN CBF h(x) / policy pi(x) forward, act, env.step, forward_graph vs the oracle
with the reference's pretrained weights.  Tolerance (SURVEY 8c): abs <= 1e-5 on h / pi
single-step (fp32 FMA path; summation order differs from the CPU), next state <= 1e-6."""
import numpy as np
import pytest
import torch

from helpers import (ENVS, oracle_env, oracle_obstacles, oracle_params, product_algo, product_env,
                     product_obstacles, random_scene)

pytestmark = pytest.mark.gpu

# strict-fp32 SIMT path: 1e-5 (SURVEY 8c).  wgmma 3xTF32 path: 3e-5 -- each of its GEMMs is within 2e-6 of |A||B| of
# float64 (tests/test_gpu_train.py), the bar here leaves room for the rounding of 3*K/8 accumulated partial products per
# output; tests/test_gpu_gnn_f64.py measures the network-level error vs float64 in units of fp32 rounding
# (tests/gnn_f64.py): measured on an H100, <= 15 units on the SIMT path and up to 260 on the tensor-core path,
# whose wgmma fp32 accumulation truncates (tests/gnn_f64.py::tc_dense reproduces it; each of its GEMMs stays within
# GEMM_BAR units of its own inputs).  Far inside the 2e-3 SURVEY 8c grants a tensor-core path.
TOL = {"simt": 1e-5, "tc": 3e-5}
CASES = [("SingleIntegrator", 8, 3, 2.0, 4), ("DoubleIntegrator", 8, 4, 2.0, 8), ("DoubleIntegrator", 48, 2, 3.0, 8),
         ("DubinsCar", 12, 3, 2.5, 6), ("LinearDrone", 10, 2, 1.5, 4)]


@pytest.mark.parametrize("env_id,N,G,area,n_obs", CASES)
def test_forward_act_step(env_id, N, G, area, n_obs, gemm_path):
    TOL_NET = TOL[gemm_path]
    from oracle.algo import act, get_cbf
    from oracle.nn import net_forward
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=2)
    env = product_env(env_id, N, area, n_obs)
    algo = product_algo(env, env_id)
    pobs = product_obstacles(env_id, obs)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    h = algo.get_cbf(graph).cpu().numpy()
    pi = algo.get_action(graph).cpu().numpy()
    a = algo.act(graph)
    u_ref = env.u_ref(graph).cpu().numpy()
    nxt = env.step(graph, a)
    fwd = env.forward_graph(graph, a)
    h_next = algo.get_cbf(fwd).cpu().numpy()
    torch.cuda.synchronize()
    graph.check_overflow()

    oenv = oracle_env(env_id, N, area, n_obs)
    ap, cp = oracle_params(env_id)
    packed = pobs.packed.cpu().numpy()
    with torch.no_grad():
        for g in range(G):
            og = oenv.sparsify(oenv.get_graph(torch.from_numpy(agent[g]), torch.from_numpy(goal[g]),
                                              oracle_obstacles(packed[g])))
            np.testing.assert_allclose(h[g], get_cbf(cp, og).numpy(), atol=TOL_NET, rtol=0)
            np.testing.assert_allclose(pi[g], net_forward(ap, og, "actor").numpy(), atol=TOL_NET, rtol=0)
            oa = act(oenv, ap, og)
            np.testing.assert_allclose(u_ref[g], oenv.u_ref(og.agent, og.goal).numpy(), atol=2e-6, rtol=3e-6)
            np.testing.assert_allclose(a[g].cpu().numpy(), oa.numpy(), atol=2 * TOL_NET + 1e-5, rtol=0)
            # env.step from the PRODUCT's action (isolates the dynamics from network rounding)
            ag = torch.from_numpy(a[g].cpu().numpy())
            og2, r, c = oenv.step(og, ag)
            np.testing.assert_allclose(nxt.graph.agent[g].cpu().numpy(), og2.agent.numpy(), atol=1e-6, rtol=0)
            np.testing.assert_allclose(nxt.reward[g].item(), r.item(), atol=1e-5, rtol=1e-5)
            np.testing.assert_allclose(nxt.cost[g].item(), c.item(), atol=1e-6)
            # forward_graph + h(g') (clip_all path, double_integrator.py:275-286, 340-354)
            ofwd = oenv.forward_graph(og, ag)
            np.testing.assert_allclose(h_next[g], get_cbf(cp, ofwd).numpy(), atol=TOL_NET, rtol=0)


def test_dense_reference_layout_equals_sparse_on_gpu_inputs(gemm_path):
    TOL_NET = TOL[gemm_path]
    """The CUDA path drops masked edges; the oracle's dense (reference) layout must agree."""
    from oracle.algo import get_cbf
    env_id, N, G, area, n_obs = "DoubleIntegrator", 8, 1, 2.0, 8
    agent, goal, obs = random_scene(env_id, N, G, area, n_obs, seed=9)
    env = product_env(env_id, N, area, n_obs)
    algo = product_algo(env, env_id)
    pobs = product_obstacles(env_id, obs)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    h = algo.get_cbf(graph).cpu().numpy()[0]
    oenv = oracle_env(env_id, N, area, n_obs)
    _, cp = oracle_params(env_id)
    dense = oenv.get_graph(torch.from_numpy(agent[0]), torch.from_numpy(goal[0]),
                           oracle_obstacles(pobs.packed.cpu().numpy()[0]))
    with torch.no_grad():
        np.testing.assert_allclose(h, get_cbf(cp, dense).numpy(), atol=TOL_NET, rtol=0)


@pytest.mark.parametrize("env_id", ["DoubleIntegrator", "LinearDrone"])
def test_cbf_contour_grid_matches_oracle(env_id):
    """test.py --cbf: get_bb_cbf (trainer/utils.py:149-168) as one batched get_cbf over 400 copies of the graph with
    tiled topology, against the oracle's 400 separate add_edge_feats + get_cbf evaluations."""
    from gcbfplus_b200.trainer.utils import get_bb_cbf
    from oracle.algo import get_bb_cbf as oracle_bb
    N, area, n_obs = 7, 1.5, 3
    agent, goal, obs = random_scene(env_id, N, 1, area, n_obs, seed=9)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 48
    pobs = product_obstacles(env_id, obs)
    graph = env.get_graph(torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs)
    algo = product_algo(env, env_id)
    xs, ys, h = get_bb_cbf(algo, env, graph.agent[0], graph.goal[0], graph.hits[0], agent_id=2)
    torch.cuda.synchronize()
    oenv = oracle_env(env_id, N, area, n_obs)
    _, cp = oracle_params(env_id)
    og = oenv.sparsify(oenv.get_graph(torch.from_numpy(agent[0]), torch.from_numpy(goal[0]),
                                      oracle_obstacles(pobs.packed.cpu().numpy()[0])))
    oxs, oys, oh = oracle_bb(oenv, cp, og, 2)
    np.testing.assert_array_equal(xs.cpu().numpy(), oxs)
    np.testing.assert_allclose(h.cpu().numpy(), oh, atol=3e-5)
    assert np.abs(oh).max() > 1e-3
