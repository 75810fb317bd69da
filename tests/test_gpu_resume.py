"""GPU: a resumed run is bit-identical to a run that was never stopped.  train.py --save-state for 4 steps against 2
steps followed by --resume: every checkpoint and the final training state (parameters, target CBF, AdamW state, both
replay buffers, the RNG states) agree to the bit, on both dense-layer paths, on one GPU and (when two are visible)
under torch.distributed.run.  load_train_state into a live trainer after a captured update() gives the same next
update as a fresh process restoring the same file (the in-place rule)."""
import os
import pickle
import socket
import subprocess
import sys

import pytest
import torch

import train
from helpers import ROOT
from gcbfplus_b200.trainer import train_state as TS

pytestmark = pytest.mark.gpu

ARGS = ["--env", "DoubleIntegrator", "-n", "8", "--area-size", "4", "--obs", "2", "--n-env-train", "4",
        "--n-env-test", "2", "--save-interval", "2", "--save-state"]


def assert_same(a, b, where="state"):
    """Recursive equality of saved states: tensors by dtype, shape and bytes, everything else by ==."""
    if isinstance(a, torch.Tensor):
        assert isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape, where
        assert a.contiguous().view(torch.uint8).equal(b.contiguous().view(torch.uint8)), where
    elif isinstance(a, dict):
        assert isinstance(b, dict) and list(a) == list(b), (where, list(a), list(b))
        for k in a:
            assert_same(a[k], b[k], f"{where}/{k}")
    elif isinstance(a, (list, tuple)):
        assert type(a) is type(b) and len(a) == len(b), where
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, f"{where}/{i}")
    else:
        assert a == b, (where, a, b)


def _run_dir(log_dir):
    runs = list(log_dir.glob("DoubleIntegrator/gcbf+/seed0_*"))
    assert len(runs) == 1, runs
    return runs[0]


def _compare_runs(full, part, world: int):
    for k in (0, 2, 4):
        for net in ("actor", "cbf"):
            a, b = (p / "models" / str(k) / f"{net}.pkl" for p in (full, part))
            assert a.read_bytes() == b.read_bytes(), f"models/{k}/{net}.pkl differs"
    for run in (full, part):
        assert sorted(os.listdir(run / TS.STATE_DIR)) == ["4", "latest"]
    for r in range(world):
        sa, sb = (torch.load(TS.state_file(str(p / TS.STATE_DIR), 4, r), weights_only=True) for p in (full, part))
        assert sa["step"] == 4 and sa["update_steps"] == 4 and sa["optim"] is not None
        # the steps after the resume drew replay samples: the buffer held more than a minibatch when they began
        assert sa["buffers"]["buffer"]["data"]["agent"].shape[0] > 2 * 256
        assert_same(sa, sb, f"rank{r}")


def test_train_py_resume_is_bit_identical(tmp_path, monkeypatch, gemm_path):
    monkeypatch.setenv("WANDB_MODE", "disabled")
    train.train(train.parse_args(ARGS + ["--steps", "4", "--log-dir", str(tmp_path / "full")]))
    train.train(train.parse_args(ARGS + ["--steps", "2", "--log-dir", str(tmp_path / "part")]))
    full, part = _run_dir(tmp_path / "full"), _run_dir(tmp_path / "part")
    assert sorted(os.listdir(part / "models")) == ["0", "2"]
    config = (part / "config.yaml").read_bytes()
    train.train(train.parse_args(["--resume", str(part), "--steps", "4"]))
    torch.cuda.synchronize()
    assert (part / "config.yaml").read_bytes() == config
    _compare_runs(full, part, world=1)
    # the checkpoints hold what an uninterrupted run trains: step 4 differs from step 2
    ck2, ck4 = (pickle.load(open(full / "models" / str(k) / "cbf.pkl", "rb")) for k in (2, 4))
    assert pickle.dumps(ck2) != pickle.dumps(ck4)


@pytest.mark.parametrize("graph_flag", ["1", "0"])
def test_restore_into_a_live_trainer_matches_a_fresh_process(tmp_path, monkeypatch, graph_flag):
    from gcbfplus_b200 import _lib
    from resume_worker import rollout_for, setup, snapshot
    monkeypatch.setenv("GCBF_TRAIN_GRAPH", "1")
    tr = setup()
    for i in range(2):
        tr.algo.update(rollout_for(tr, i), i)
        tr.update_steps += 1
    state = str(tmp_path / "rank0.pt")
    TS.save_train_state(tr, state, 2)
    tr.algo.update(rollout_for(tr, 2), 2)          # the live objects move on through a captured update
    torch.cuda.synchronize()
    assert TS.load_train_state(tr, state) == 2
    monkeypatch.setenv("GCBF_TRAIN_GRAPH", graph_flag)
    live = snapshot(tr, tr.algo.update(rollout_for(tr, 2), 2))
    out = str(tmp_path / "fresh.pt")
    env = dict(os.environ, GCBF_TENSOR_CORES="1" if _lib.USE_TC else "0")
    proc = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "resume_worker.py"), state, out], env=env,
                          capture_output=True, text=True, timeout=600)
    assert proc.returncode == 0, proc.stdout[-3000:] + proc.stderr[-3000:]
    fresh = torch.load(out, weights_only=True)
    assert live["buffers"]["buffer"]["data"] is not None
    assert_same(live, fresh)


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _torchrun(argv, timeout=900):
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr",
           "127.0.0.1", "--master-port", str(_free_port()), os.path.join(ROOT, "train.py")] + argv
    proc = subprocess.Popen(cmd, cwd=ROOT, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                            env=dict(os.environ, WANDB_MODE="disabled"), start_new_session=True)
    try:
        out, _ = proc.communicate(timeout=timeout)
    except subprocess.TimeoutExpired:
        import signal
        os.killpg(proc.pid, signal.SIGKILL)                 # exactly the process group this test started
        out, _ = proc.communicate()
        raise AssertionError("train.py under torch.distributed.run timed out; output so far:\n" + out[-4000:])
    assert proc.returncode == 0, out[-4000:]


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs >= 2 GPUs")
def test_two_gpu_resume_is_bit_identical(tmp_path):
    _torchrun(ARGS + ["--steps", "4", "--log-dir", str(tmp_path / "full")])
    _torchrun(ARGS + ["--steps", "2", "--log-dir", str(tmp_path / "part")])
    part = _run_dir(tmp_path / "part")
    _torchrun(["--resume", str(part), "--steps", "4"])
    _compare_runs(_run_dir(tmp_path / "full"), part, world=2)
