"""Training state: everything that decides the rest of a `Trainer.train` run, saved beside a model checkpoint and
restored in place, so that a stopped run continues with the bits it would have produced had it never stopped
(DESIGN §4.8).

Layout of `<run>/train_state/`:
    <k>/rank<r>.pt   rank r's state at the top of step k: `torch.save` of CPU tensors and plain Python values
    latest           JSON record of the last complete state: its step and the context a resume must match
Only the latest complete state is kept.  Every file is written under a temporary name and renamed, and `latest` moves
to step k only after every rank has written its step-k file, so a stop partway through a save leaves the previous
state complete and usable.
"""
from __future__ import annotations

import json
import os
import warnings
from typing import Optional

import numpy as np
import torch

from .. import _lib
from .. import dist as gdist
from ..algo.train import init_update_state
from ..utils import jrandom as jr

FORMAT = 1
STATE_DIR = "train_state"      # under the run directory
# TrainState tensors that carry over between updates (the rest is per-minibatch scratch, rewritten before it is read)
OPTIM_FIELDS = ("m_cbf", "v_cbf", "step_cbf", "m_act", "v_act", "step_act", "overflow")
# context a resumed run must share with the saved one: (key, what the message calls it)
REQUIRED = (("world_size", "world size (number of ranks)"),
            ("threefry_partitionable", "threefry layout (GCBF_THREEFRY_PARTITIONABLE)"),
            ("use_tc", "dense-layer path (GCBF_TENSOR_CORES)"))


def _world_rank():
    world = gdist.world_size()
    return world, (gdist.dist.get_rank() if world > 1 else 0)


def run_context(world: int) -> dict:
    """The context of this process that a resume must match (REQUIRED)."""
    return {"world_size": int(world), "threefry_partitionable": bool(jr.PARTITIONABLE), "use_tc": bool(_lib.USE_TC)}


def _device_context(device: torch.device) -> dict:
    """GPU model and SM count: the determinism contract holds on the same GPU model (the SM count sets split counts)."""
    if device.type != "cuda":
        return {"gpu_name": None, "sm_count": None}
    p = torch.cuda.get_device_properties(device)
    return {"gpu_name": p.name, "sm_count": int(p.multi_processor_count)}


def check_context(saved: dict, current: dict) -> None:
    """Raise ValueError naming every REQUIRED entry in which `saved` and `current` differ."""
    bad = [f"{what}: saved {saved.get(k)!r}, this run {current[k]!r}"
           for k, what in REQUIRED if saved.get(k) != current[k]]
    if bad:
        raise ValueError("the saved training state does not match this run: " + "; ".join(bad))


def state_file(state_dir: str, step: int, rank: int) -> str:
    return os.path.join(state_dir, str(step), f"rank{rank}.pt")


def _atomic_write(path: str, write) -> None:
    tmp = path + ".tmp"
    with open(tmp, "wb") as f:
        write(f)
        f.flush()
        os.fsync(f.fileno())
    os.replace(tmp, path)


def _cpu(t: torch.Tensor) -> torch.Tensor:
    return t.detach().to("cpu", copy=True)


def _buffer_state(buf) -> Optional[dict]:
    if buf is None:
        return None
    return {"data": None if buf._data is None else {k: _cpu(v) for k, v in buf._data.items()}, "T": int(buf._T)}


def state_dict(trainer, step: int) -> dict:
    """CPU copies of rank-local training state at the top of step `step` (before its rollout)."""
    algo, env = trainer.algo, trainer.env
    world, rank = _world_rank()
    ts = algo._trainer_state
    np_state = np.random.get_state()
    return {
        "format": FORMAT, "step": int(step), "update_steps": int(trainer.update_steps),
        "key": [int(x) for x in trainer.key],
        "context": dict(run_context(world), rank=rank, **_device_context(env.device)),
        "params": {"cbf": _cpu(algo.cbf_params.flat), "cbf_tgt": _cpu(algo.cbf_tgt_params.flat),
                   "actor": _cpu(algo.actor_net_params.flat)},
        "optim": None if ts is None else {k: _cpu(getattr(ts, k)) for k in OPTIM_FIELDS},
        "buffers": {name: _buffer_state(getattr(algo, name, None)) for name in ("buffer", "unsafe_buffer")},
        "algo_rng": algo.rng.bit_generator.state,
        "np_rng": [np_state[0], torch.from_numpy(np_state[1].astype(np.int64)), int(np_state[2]), int(np_state[3]),
                   float(np_state[4])],
        "edge_cap_per_agent": int(env.edge_cap_per_agent),
    }


def save_train_state(trainer, path: str, step: int) -> None:
    """Write this rank's training state at the top of step `step` to `path` (temporary file, then rename)."""
    sd = state_dict(trainer, step)
    _atomic_write(path, lambda f: torch.save(sd, f))


def _copy_into(dst: torch.Tensor, src: torch.Tensor, what: str) -> None:
    if dst.shape != src.shape or dst.dtype != src.dtype:
        raise ValueError(f"{what}: saved {tuple(src.shape)} {src.dtype}, this run {tuple(dst.shape)} {dst.dtype}")
    dst.copy_(src)


def load_train_state(trainer, path: str) -> int:
    """Restore the state `save_train_state` wrote into a live trainer, its algo and its env; returns the step to start
    at.  Parameters and optimizer state are copied into the existing tensors (the rollout engines and captured
    minibatch graphs hold raw device pointers to them); TrainState and the replay buffers are built first where update()
    would build them lazily."""
    sd = torch.load(path, map_location="cpu", weights_only=True, mmap=True)
    if sd.get("format") != FORMAT:
        raise ValueError(f"{path}: training state format {sd.get('format')!r}, this version reads {FORMAT}")
    algo, env = trainer.algo, trainer.env
    world, rank = _world_rank()
    ctx = sd["context"]
    check_context(ctx, run_context(world))
    if ctx["rank"] != rank:
        raise ValueError(f"{path} holds rank {ctx['rank']}'s state, this process is rank {rank}")
    here = _device_context(env.device)
    if (ctx["gpu_name"], ctx["sm_count"]) != (here["gpu_name"], here["sm_count"]):
        warnings.warn(f"the training state was saved on {ctx['gpu_name']} ({ctx['sm_count']} SMs), this run is on "
                      f"{here['gpu_name']} ({here['sm_count']} SMs): the run continues, but it is not promised to be "
                      "bit-identical to an uninterrupted run (determinism holds on one GPU model)", RuntimeWarning)
    for name, p in (("cbf", algo.cbf_params), ("cbf_tgt", algo.cbf_tgt_params), ("actor", algo.actor_net_params)):
        _copy_into(p.flat, sd["params"][name], f"params/{name}")
    init_update_state(algo)
    ts = algo._trainer_state
    for k in OPTIM_FIELDS:
        if sd["optim"] is None:          # saved before the first update: a fresh TrainState is all zeros
            getattr(ts, k).zero_()
        else:
            _copy_into(getattr(ts, k), sd["optim"][k], f"optim/{k}")
    for name in ("buffer", "unsafe_buffer"):
        buf, saved = getattr(algo, name), sd["buffers"][name]
        # the buffers are not captured anywhere: every append replaces their arrays, so new ones are fine here
        buf._data = None if saved is None or saved["data"] is None else \
            {k: v.to(env.device, copy=True) for k, v in saved["data"].items()}
        buf._T = 1 if saved is None else saved["T"]
    algo.rng.bit_generator.state = sd["algo_rng"]
    name, keys, pos, has_gauss, cached = sd["np_rng"]
    np.random.set_state((name, keys.numpy().astype(np.uint32), pos, has_gauss, cached))
    trainer.key = np.array(sd["key"], dtype=np.uint32)
    trainer.update_steps = sd["update_steps"]
    trainer.start_step = sd["step"]
    env.edge_cap_per_agent = sd["edge_cap_per_agent"]
    return sd["step"]


def _barrier(world: int) -> None:
    if world > 1:
        gdist.dist.barrier()


def save_run_state(trainer, state_dir: str, step: int) -> None:
    """Every rank writes `<step>/rank<r>.pt`; after a barrier rank 0 points `latest` at step; after a second barrier
    every rank removes its files of earlier states."""
    world, rank = _world_rank()
    os.makedirs(os.path.join(state_dir, str(step)), exist_ok=True)
    save_train_state(trainer, state_file(state_dir, step, rank), step)
    _barrier(world)
    if rank == 0:
        rec = dict(format=FORMAT, step=int(step), **run_context(world), **_device_context(trainer.env.device))
        _atomic_write(os.path.join(state_dir, "latest"), lambda f: f.write(json.dumps(rec).encode()))
    _barrier(world)
    for d in os.listdir(state_dir):
        if d.isdigit() and int(d) != step:
            old = state_file(state_dir, int(d), rank)
            for p in (old, old + ".tmp"):
                if os.path.exists(p):
                    os.remove(p)
            try:
                os.rmdir(os.path.join(state_dir, d))    # the last rank to clear its files removes the directory
            except OSError:
                pass


def check_resume(state_dir: str, world: int) -> dict:
    """The `latest` record of a complete training state in `state_dir` that a run of `world` ranks in this process's
    context may resume from; ValueError otherwise.  Reads only small files: no device work."""
    rec_path = os.path.join(state_dir, "latest")
    try:
        with open(rec_path) as f:
            rec = json.load(f)
    except (OSError, ValueError):
        raise ValueError(f"no complete training state in {state_dir} (train.py --save-state writes one)") from None
    if rec.get("format") != FORMAT or "step" not in rec:
        raise ValueError(f"{rec_path}: not a training state record of format {FORMAT}")
    missing = [r for r in range(int(rec.get("world_size", 0)))
               if not os.path.isfile(state_file(state_dir, rec["step"], r))]
    if missing:
        raise ValueError(f"no complete training state in {state_dir}: {rec_path} names step {rec['step']}, "
                         f"rank files missing: {missing}")
    check_context(rec, run_context(world))
    return rec
