"""GPU determinism: on one GPU, the same inputs give the same bits, run after run -- the canonical edge layout of the
graph build, the train step's fixed-order reductions (both dense-layer paths), the QP labels, update() on the captured
and the eager path, and train.py end to end."""
import pickle

import numpy as np
import pytest
import torch

from helpers import (edge_sets_oracle, edge_sets_product, oracle_env, oracle_obstacles, product_algo,
                     product_env, product_obstacles, random_scene)

pytestmark = pytest.mark.gpu

# (env, N, B, area, n_obs): sizes where the dW GEMMs split the rows over many CTAs
LAYOUT_CASES = [("SingleIntegrator", 64, 8, 3.0, 4), ("DoubleIntegrator", 128, 32, 5.0, 6),
                ("DubinsCar", 64, 8, 3.2, 4), ("LinearDrone", 64, 8, 2.2, 3)]
TRAIN_CASES = [("DoubleIntegrator", 128, 32, 5.0, 6), ("LinearDrone", 64, 16, 2.2, 3), ("DubinsCar", 64, 16, 3.2, 4)]
GRAPH_FIELDS = ("row_start", "row_deg", "edge_recv", "edge_src", "hits", "counters")


def _scene(env_id, N, B, area, n_obs, seed=11):
    agent, goal, obs = random_scene(env_id, N, B, area, n_obs, seed, vel_scale=0.45)
    env = product_env(env_id, N, area, n_obs)
    env.edge_cap_per_agent = 64
    pobs = product_obstacles(env_id, obs)
    return env, torch.from_numpy(agent).cuda(), torch.from_numpy(goal).cuda(), pobs


def _bits(t: torch.Tensor) -> bytes:
    return t.detach().contiguous().cpu().numpy().tobytes()


@pytest.mark.parametrize("env_id,N,B,area,n_obs", LAYOUT_CASES)
def test_graph_layout_is_canonical_and_repeatable(env_id, N, B, area, n_obs):
    env, agent, goal, pobs = _scene(env_id, N, B, area, n_obs)
    g1 = env.get_graph(agent, goal, pobs)
    g2 = env.get_graph(agent, goal, pobs)
    torch.cuda.synchronize()
    g1.check_overflow()
    deg = g1.row_deg.long()
    start = torch.cat([torch.zeros(1, dtype=torch.long, device=deg.device), deg.cumsum(0)[:-1]])
    assert torch.equal(g1.row_start.long(), start)
    total = int(deg.sum())
    assert int(g1.counters[0]) == total
    recv = g1.edge_recv[:total].long()
    assert torch.equal(recv, torch.repeat_interleave(torch.arange(B * N, device=deg.device), deg))
    for f in GRAPH_FIELDS:
        assert _bits(getattr(g1, f)) == _bits(getattr(g2, f)), f
    # every row still holds exactly what the build writes for it
    oenv = oracle_env(env_id, N, area, n_obs)
    packed = pobs.packed.cpu().numpy()
    a_np, g_np = agent.cpu().numpy(), goal.cpu().numpy()
    for g in (0, B - 1):
        og = oenv.sparsify(oenv.get_graph(torch.from_numpy(a_np[g]), torch.from_numpy(g_np[g]),
                                          oracle_obstacles(packed[g])))
        assert edge_sets_product(g1, g, N) == edge_sets_oracle(og, N, env.n_hits)


def _train_setup(env_id, N, B, area, n_obs):
    env, agent, goal, pobs = _scene(env_id, N, B, area, n_obs, seed=21)
    algo = product_algo(env, env_id, seed=3)
    algo.loss_action_coef, algo.loss_h_dot_coef = 0.05, 0.3
    graph = env.get_graph(agent, goal, pobs)
    rng = np.random.default_rng(5)
    unsafe = env.unsafe_mask(graph)
    safe = (~unsafe) & torch.from_numpy(rng.uniform(size=(B, N)) < 0.6).cuda()
    u_qp = env.u_ref(graph) + torch.from_numpy(rng.normal(0, 0.1, size=(B, N, env.action_dim)).astype(np.float32)).cuda()
    return env, algo, agent, goal, pobs, safe, unsafe, u_qp


@pytest.mark.parametrize("env_id,N,B,area,n_obs", TRAIN_CASES)
def test_train_step_is_bit_identical(env_id, N, B, area, n_obs, gemm_path):
    from gcbfplus_b200.algo.train import train_minibatch
    env, algo, agent, goal, pobs, safe, unsafe, u_qp = _train_setup(env_id, N, B, area, n_obs)
    runs = []
    for _ in range(5):
        graph = env.get_graph(agent, goal, pobs)       # a fresh build each time: the layout must not vary either
        ts = train_minibatch(algo, graph, safe, unsafe, u_qp, apply=False)
        torch.cuda.synchronize()
        graph.check_overflow()
        runs.append((_bits(ts.grad_cbf), _bits(ts.grad_act), _bits(ts.stats)))
    assert torch.isfinite(ts.grad_cbf).all() and torch.isfinite(ts.grad_act).all()
    assert float(ts.grad_cbf.abs().max()) > 0 and float(ts.grad_act.abs().max()) > 0
    for r in runs[1:]:
        assert r[0] == runs[0][0], "grad_cbf differs between runs"
        assert r[1] == runs[0][1], "grad_actor differs between runs"
        assert r[2] == runs[0][2], "stats differ between runs"


def test_qp_labels_are_bit_identical(gemm_path):
    from gcbfplus_b200.algo.train import qp_labels
    env, agent, goal, pobs = _scene("DoubleIntegrator", 64, 16, 4.0, 4, seed=9)
    algo = product_algo(env, "DoubleIntegrator", seed=0)
    outs = []
    for _ in range(2):
        graph = env.get_graph(agent, goal, pobs)
        u, aux, iters = qp_labels(algo, graph, with_aux=True)
        torch.cuda.synchronize()
        graph.check_overflow()
        outs.append((_bits(u), _bits(aux), _bits(iters)))
    assert outs[0] == outs[1]


def _update_once(env, rollout, graph_flag, monkeypatch):
    monkeypatch.setenv("GCBF_TRAIN_GRAPH", graph_flag)
    np.random.seed(0)
    algo = product_algo(env, "DoubleIntegrator", seed=0)
    algo.batch_size, algo.inner_epoch, algo.lr_cbf, algo.lr_actor = 48, 2, 1e-3, 1e-3
    info = algo.update(rollout, 0)
    torch.cuda.synchronize()
    ts = algo._trainer_state
    state = [algo.cbf_params.flat, algo.actor_params.flat, algo.cbf_tgt_params.flat, ts.m_cbf, ts.v_cbf, ts.m_act,
             ts.v_act, ts.step_cbf, ts.step_act]
    return [_bits(t) for t in state], info


def test_update_is_bit_identical_captured_and_eager(monkeypatch):
    from gcbfplus_b200.trainer.rollout import RolloutEngine
    env = product_env("DoubleIntegrator", 8, 3.0, 4)
    algo0 = product_algo(env, "DoubleIntegrator", seed=0)
    eng = RolloutEngine(env, 3, T=32, n_obs=4)
    eng.set_params(algo0.actor_params)
    g0 = env.reset(5, n_envs=3)
    eng.set_initial(g0.agent, g0.goal, g0.obstacle)
    eng.run()
    rollout = eng.result()
    a_state, a_info = _update_once(env, rollout, "1", monkeypatch)
    b_state, b_info = _update_once(env, rollout, "1", monkeypatch)
    c_state, c_info = _update_once(env, rollout, "0", monkeypatch)
    names = ("cbf", "actor", "cbf_tgt", "m_cbf", "v_cbf", "m_act", "v_act", "step_cbf", "step_act")
    for n, a, b, c in zip(names, a_state, b_state, c_state):
        assert a == b, f"{n}: two captured runs differ"
        assert a == c, f"{n}: captured and eager paths differ"
    assert a_info == b_info
    assert a_info == c_info


def test_train_py_checkpoints_are_bit_identical(tmp_path, monkeypatch):
    import train as train_mod
    monkeypatch.setenv("WANDB_MODE", "disabled")
    runs = []
    for i in range(2):
        log_dir = tmp_path / f"run{i}"
        args = train_mod.build_parser(train_mod.FLAGS).parse_args(
            ["--env", "DoubleIntegrator", "-n", "8", "--area-size", "4", "--obs", "2", "--seed", "3", "--steps", "3",
             "--n-env-train", "4", "--n-env-test", "2", "--eval-interval", "1", "--save-interval", "1",
             "--lr-actor", "1e-3", "--lr-cbf", "1e-3", "--log-dir", str(log_dir)])
        train_mod.train(args)
        torch.cuda.synchronize()
        models = sorted(log_dir.glob("DoubleIntegrator/gcbf+/seed3_*/models"))
        assert len(models) == 1, models
        ck = {}
        for step_dir in sorted(models[0].iterdir(), key=lambda p: int(p.name)):
            for net in ("cbf", "actor"):
                ck[(int(step_dir.name), net)] = pickle.load(open(step_dir / f"{net}.pkl", "rb"))
        runs.append(ck)
    # a checkpoint per step, each written before that step's update: step 3 holds the result of three updates
    assert set(runs[0]) == set(runs[1]) and {s for s, _ in runs[0]} == {0, 1, 2, 3}, sorted(runs[0])

    def leaves(tree, prefix=""):
        if isinstance(tree, dict):
            for k in sorted(tree):
                yield from leaves(tree[k], f"{prefix}/{k}")
        else:
            yield prefix, np.asarray(tree)

    for key in runs[0]:
        la, lb = list(leaves(runs[0][key])), list(leaves(runs[1][key]))
        assert [n for n, _ in la] == [n for n, _ in lb]
        for (n, x), (_, y) in zip(la, lb):
            assert x.dtype == y.dtype and x.shape == y.shape and x.tobytes() == y.tobytes(), (key, n)
