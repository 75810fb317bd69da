"""CPU: the training state of trainer/train_state.py and train.py --resume.  The rejections of a run that cannot
resume (no state, an extra flag, fewer --steps, another world size / threefry layout / dense-layer path) happen before
any directory or file is written; the replay buffers, the minibatch permutation generator and NumPy's global RNG
round-trip through save / load (the next samples are identical); a two-rank gloo save writes one file per rank and
keeps only the latest state.  End-to-end bit identity is tests/test_gpu_resume.py."""
import json
import os
import shutil
import socket
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

import train
from gcbfplus_b200.algo.train import init_update_state
from gcbfplus_b200.trainer import train_state as TS
from gcbfplus_b200.utils import jrandom as jr

N, T = 4, 3


def _cpu_trainer(seed: int):
    """The pieces of a Trainer / GCBFPlus the training state reads and writes, on the CPU."""
    from gcbfplus_b200.algo.params import NetParams
    env = SimpleNamespace(device=torch.device("cpu"), edge_cap_per_agent=16)
    cbf = NetParams(4, 1, "cbf", device="cpu").init_xavier(2 * seed + 1)
    algo = SimpleNamespace(_env=env, buffer_size=6, rng=np.random.default_rng(seed + 1), _trainer_state=None,
                           cbf_params=cbf, cbf_tgt_params=cbf.clone(),
                           actor_net_params=NetParams(4, 2, "actor", device="cpu").init_xavier(2 * seed + 2))
    return SimpleNamespace(env=env, algo=algo, key=jr.PRNGKey(seed), update_steps=0, start_step=0)


def _train_a_little(tr, seed: int, n_rollouts: int = 9):
    """What updates leave behind: full (wrapped) replay buffers, moved optimizer state and parameters, advanced RNGs."""
    rng = np.random.default_rng(seed)
    algo = tr.algo
    init_update_state(algo)
    for _ in range(n_rollouts):
        f = lambda *s: torch.from_numpy(rng.normal(size=s).astype(np.float32))
        new = {"agent": f(T, N, 4), "hits": f(T, N, 32, 2), "goal": f(T, N, 4),
               "safe": torch.from_numpy((rng.uniform(size=(T, N)) < 0.5).astype(np.uint8)),
               "unsafe": torch.from_numpy((rng.uniform(size=(T, N)) < 0.3).astype(np.uint8))}
        algo.buffer.append_rollouts(new, 1, T)
        algo.unsafe_buffer.append_graphs(new, new["unsafe"].any(dim=-1))
    ts = algo._trainer_state
    for k in ("m_cbf", "v_cbf", "m_act", "v_act"):
        getattr(ts, k).copy_(torch.from_numpy(rng.normal(size=getattr(ts, k).shape).astype(np.float32)))
    ts.step_cbf.fill_(n_rollouts)
    ts.step_act.fill_(n_rollouts)
    ts.overflow.fill_(1)
    for p in (algo.cbf_params, algo.cbf_tgt_params, algo.actor_net_params):
        p.flat.add_(0.01)
    algo.rng.permutation(50)
    np.random.seed(seed + 100)
    np.random.randint(0, 9, 17)
    _, tr.key = jr.split(tr.key)
    tr.update_steps = n_rollouts
    tr.env.edge_cap_per_agent = 32


def _next_draws(tr):
    """What the next update() would draw: replay samples (NumPy's global RNG) and a minibatch permutation (algo.rng)."""
    algo = tr.algo
    return {"memory": algo.buffer.sample_rollouts(5), "unsafe_memory": algo.unsafe_buffer.sample_graphs(7),
            "perm": algo.rng.permutation(40), "np": np.random.randint(0, 1000, 8)}


def _equal_draws(a, b):
    for k in ("memory", "unsafe_memory"):
        assert a[k].keys() == b[k].keys()
        for f in a[k]:
            assert a[k][f].dtype == b[k][f].dtype and torch.equal(a[k][f], b[k][f]), (k, f)
    assert np.array_equal(a["perm"], b["perm"]) and np.array_equal(a["np"], b["np"])


def test_state_round_trips_through_save_and_load(tmp_path):
    a = _cpu_trainer(0)
    _train_a_little(a, seed=1)
    assert a.algo.buffer.length == 6 * T and a.algo.unsafe_buffer.length == 3   # both buffers wrapped
    path = str(tmp_path / "rank0.pt")
    TS.save_train_state(a, path, step=4)
    assert not os.path.exists(path + ".tmp")
    want = _next_draws(a)
    b = _cpu_trainer(7)                      # other seeds: every piece below must come from the file
    np.random.seed(5)
    assert TS.load_train_state(b, path) == 4
    assert b.start_step == 4 and b.update_steps == a.update_steps and b.env.edge_cap_per_agent == 32
    assert b.key.dtype == np.uint32 and np.array_equal(b.key, a.key)
    for n in ("cbf_params", "cbf_tgt_params", "actor_net_params"):
        assert torch.equal(getattr(b.algo, n).flat, getattr(a.algo, n).flat), n
    for k in TS.OPTIM_FIELDS:
        assert torch.equal(getattr(b.algo._trainer_state, k), getattr(a.algo._trainer_state, k)), k
    _equal_draws(_next_draws(b), want)


def test_state_saved_before_the_first_update_empties_a_used_trainer(tmp_path):
    """A state from step 0 (no TrainState, no buffers yet) loaded into a trainer that has trained: zero optimizer state,
    empty buffers, as update() would build them."""
    a = _cpu_trainer(0)
    path = str(tmp_path / "rank0.pt")
    TS.save_train_state(a, path, step=0)
    b = _cpu_trainer(0)
    _train_a_little(b, seed=2)
    assert TS.load_train_state(b, path) == 0
    ts = b.algo._trainer_state
    assert all(int(torch.count_nonzero(getattr(ts, k))) == 0 for k in TS.OPTIM_FIELDS)
    assert b.algo.buffer.length == 0 and b.algo.unsafe_buffer.length == 0
    assert torch.equal(b.algo.cbf_params.flat, a.algo.cbf_params.flat) and b.env.edge_cap_per_agent == 16
    assert b.algo.rng.bit_generator.state == a.algo.rng.bit_generator.state


@pytest.mark.parametrize("key,value,name", [("world_size", 2, "world size"),
                                            ("threefry_partitionable", not jr.PARTITIONABLE, "GCBF_THREEFRY_PARTITIONABLE"),
                                            ("use_tc", None, "GCBF_TENSOR_CORES")])
def test_load_refuses_a_state_of_another_context(tmp_path, key, value, name):
    from gcbfplus_b200 import _lib
    a = _cpu_trainer(0)
    path = str(tmp_path / "rank0.pt")
    TS.save_train_state(a, path, step=2)
    sd = torch.load(path, weights_only=True)
    sd["context"][key] = (not _lib.USE_TC) if key == "use_tc" else value
    torch.save(sd, path)
    b = _cpu_trainer(3)
    before = b.algo.cbf_params.flat.clone()
    with pytest.raises(ValueError, match=name):
        TS.load_train_state(b, path)
    assert torch.equal(b.algo.cbf_params.flat, before)


# ------------------------------------------------------------------------------------ train.py --resume
def _run_dir(tmp_path, steps: int = 4):
    """A run directory as train.py leaves it: config.yaml, models/."""
    run = tmp_path / "run"
    os.makedirs(run / "models")
    args = train.build_parser(train.FLAGS).parse_args(
        ["--env", "DoubleIntegrator", "-n", "8", "--area-size", "4", "--obs", "2", "--n-env-train", "4",
         "--n-env-test", "2", "--save-interval", "2", "--steps", str(steps), "--save-state", "--log-dir", str(tmp_path)])
    train.write_config(str(run), args, {"batch_size": 256})
    return run


def _save_state(run, step: int):
    tr = _cpu_trainer(0)
    TS.save_run_state(tr, str(run / TS.STATE_DIR), step)


def _tree(root):
    return sorted((os.path.relpath(os.path.join(d, f), root), os.path.getmtime(os.path.join(d, f)))
                  for d, _, fs in os.walk(root) for f in fs) + sorted(d for d, _, _ in os.walk(root))


def _rejected(tmp_path, argv, match):
    before = _tree(tmp_path)
    with pytest.raises(SystemExit, match=match):
        train.train(train.parse_args(argv))
    assert _tree(tmp_path) == before, "a rejected --resume wrote to the file system"


def test_config_records_the_run_not_the_invocation(tmp_path):
    import yaml
    run = _run_dir(tmp_path)
    cfg = yaml.load(open(run / "config.yaml"), Loader=yaml.UnsafeLoader)
    assert cfg.num_agents == 8 and cfg.steps == 4 and cfg.batch_size == 256
    assert not hasattr(cfg, "resume") and not hasattr(cfg, "save_state")


def test_resume_takes_every_flag_from_the_run(tmp_path):
    run = _run_dir(tmp_path)
    args = train.parse_args(["--resume", str(run)])          # no --area-size: it comes from config.yaml
    assert (args.env, args.num_agents, args.area_size, args.obs, args.steps) == ("DoubleIntegrator", 8, 4.0, 2, 4)
    assert args.resume == str(run) and args.save_state
    assert train.parse_args(["--resume", str(run), "--steps", "9"]).steps == 9


@pytest.mark.parametrize("extra", [["--seed", "1"], ["--area-size", "4"], ["--save-state"], ["--debug"],
                                   ["-n", "8"], ["--lr-cbf", "3e-5"]])
def test_resume_rejects_any_other_flag(tmp_path, extra):
    run = _run_dir(tmp_path)
    _save_state(run, 2)
    flag = extra[0] if extra[0] != "-n" else "--num-agents"
    before = _tree(tmp_path)
    with pytest.raises(SystemExit, match=flag):
        train.parse_args(["--resume", str(run), "--steps", "6"] + extra)
    assert _tree(tmp_path) == before


def test_resume_without_a_state_is_rejected_before_any_write(tmp_path):
    run = _run_dir(tmp_path)
    _rejected(tmp_path, ["--resume", str(run)], "no complete training state")
    with pytest.raises(SystemExit, match="config.yaml"):
        train.parse_args(["--resume", str(tmp_path / "missing")])
    assert not (tmp_path / "missing").exists()


def test_resume_with_a_missing_rank_file_is_rejected(tmp_path):
    run = _run_dir(tmp_path)
    _save_state(run, 2)
    os.remove(TS.state_file(str(run / TS.STATE_DIR), 2, 0))
    _rejected(tmp_path, ["--resume", str(run)], "rank files missing")


def test_resume_with_fewer_steps_is_rejected(tmp_path):
    run = _run_dir(tmp_path, steps=4)
    _save_state(run, 4)
    _rejected(tmp_path, ["--resume", str(run), "--steps", "2"], "below the saved step 4")


@pytest.mark.parametrize("key,name", [("world_size", "world size"),
                                      ("threefry_partitionable", "GCBF_THREEFRY_PARTITIONABLE"),
                                      ("use_tc", "GCBF_TENSOR_CORES")])
def test_resume_with_another_context_is_rejected(tmp_path, key, name):
    run = _run_dir(tmp_path)
    _save_state(run, 2)
    state_dir = run / TS.STATE_DIR
    rec = json.loads((state_dir / "latest").read_text())
    rec[key] = 2 if key == "world_size" else not rec[key]
    (state_dir / "latest").write_text(json.dumps(rec))
    if key == "world_size":    # a complete two-rank state
        shutil.copy(TS.state_file(str(state_dir), 2, 0), TS.state_file(str(state_dir), 2, 1))
    _rejected(tmp_path, ["--resume", str(run)], name)


# ------------------------------------------------------------------------------------ two ranks (gloo)
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, state_dir, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world),
                      LOCAL_RANK=str(rank))
    torch.set_num_threads(1)
    from gcbfplus_b200 import dist as gd
    gd.init_from_env(backend="gloo")
    tr = _cpu_trainer(rank)
    TS.save_run_state(tr, state_dir, 2)
    _train_a_little(tr, seed=10 + rank)
    TS.save_run_state(tr, state_dir, 4)
    want = _next_draws(tr)
    fresh = _cpu_trainer(9)
    step = TS.load_train_state(fresh, TS.state_file(state_dir, 4, rank))
    _equal_draws(_next_draws(fresh), want)
    torch.save({"step": step, "cbf": fresh.algo.cbf_params.flat}, f"{out}.{rank}")
    dist.destroy_process_group()


def test_two_ranks_write_one_state_file_each_and_keep_only_the_latest(tmp_path):
    state_dir = str(tmp_path / TS.STATE_DIR)
    out = str(tmp_path / "res")
    mp.spawn(_worker, args=(2, _free_port(), state_dir, out), nprocs=2, join=True)
    assert sorted(os.listdir(state_dir)) == ["4", "latest"]
    assert sorted(os.listdir(os.path.join(state_dir, "4"))) == ["rank0.pt", "rank1.pt"]
    rec = json.loads(open(os.path.join(state_dir, "latest")).read())
    assert rec["step"] == 4 and rec["world_size"] == 2
    res = [torch.load(f"{out}.{r}", weights_only=True) for r in range(2)]
    assert all(r["step"] == 4 for r in res)
    assert not torch.equal(res[0]["cbf"], res[1]["cbf"])      # each rank restored its own file
    for r in range(2):
        sd = torch.load(TS.state_file(state_dir, 4, r), weights_only=True)
        assert sd["context"]["rank"] == r and sd["context"]["world_size"] == 2
    # a one-rank run cannot resume it
    with pytest.raises(ValueError, match="world size"):
        TS.check_resume(state_dir, 1)
