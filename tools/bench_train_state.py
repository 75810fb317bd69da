#!/usr/bin/env python
"""Cost of saving and restoring the training state (trainer/train_state.py, train.py --save-state / --resume) with
both replay buffers full, at configs[2] shapes on one GPU.

    python tools/bench_train_state.py [--rollouts 512] [--T 256] [--dir /tmp] [--repeats 2]

Builds a DoubleIntegrator n = 512, obs 8 GCBF+ trainer and fills its replay buffer with --rollouts rollouts of T
graphs (default: the capacity, buffer_size 512 x the 256-step episode) and its unsafe-graph buffer to its capacity of
256 graphs, without training: the arrays are written directly, with values drawn on the device.  Then times
save_train_state (device-to-host copies, torch.save, fsync, rename) and load_train_state (torch.load, host-to-device
copies) --repeats times.  The load reads a file that was just written, so it comes from the page cache, not the disk.
Prints one JSON line: the file's bytes, the bytes computed from shapes, the seconds of every repeat and the card and
its power limit.  Writes only the state file, under --dir, and removes it."""
import argparse
import json
import os
import shutil
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from bench import CONFIGS  # noqa: E402


def _mem_available() -> int:
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rollouts", type=int, default=512, help="stored rollouts (the buffer holds buffer_size = 512)")
    ap.add_argument("--T", type=int, default=256, help="graphs per stored rollout (the episode length)")
    ap.add_argument("--dir", type=str, default=tempfile.gettempdir(), help="where the state file is written")
    ap.add_argument("--repeats", type=int, default=2)
    args = ap.parse_args()
    import torch
    from gcbfplus_b200 import _lib
    from gcbfplus_b200.algo import make_algo
    from gcbfplus_b200.algo.train import init_update_state
    from gcbfplus_b200.env import make_env
    from gcbfplus_b200.trainer.train_state import load_train_state, save_train_state
    from gcbfplus_b200.trainer.trainer import Trainer
    if not torch.cuda.is_available():
        raise RuntimeError("tools/bench_train_state.py needs a CUDA device: the product path has no CPU fallback")
    _lib.load(build_if_missing=False)
    cfg = CONFIGS[3]
    N = cfg["N"]
    env = make_env(cfg["env"], N, area_size=cfg["area"], num_obs=cfg["obs"], device="cuda")
    algo = make_algo("gcbf+", env=env, node_dim=env.node_dim, edge_dim=env.edge_dim, state_dim=env.state_dim,
                     action_dim=env.action_dim, n_agents=N, buffer_size=512, seed=0)
    params = {"run_name": "bench", "training_steps": 0, "eval_interval": 1, "eval_epi": 1, "save_interval": 1}
    tr = Trainer(env, env, algo, n_env_train=cfg["envs_total"], n_env_test=1, log_dir="", seed=0, params=params,
                 save_log=False)
    init_update_state(algo)
    rows = {"buffer": min(args.rollouts, algo.buffer_size) * args.T, "unsafe_buffer": algo.buffer_size // 2}
    shapes = {"agent": (N, env.state_dim), "hits": (N, env.n_hits, env.pos_dim), "goal": (N, env.state_dim),
              "safe": (N,), "unsafe": (N,)}
    per_graph = sum(int(torch.tensor(s).prod()) * (1 if k in ("safe", "unsafe") else 4) for k, s in shapes.items())
    computed = per_graph * sum(rows.values())
    free_disk, free_ram = shutil.disk_usage(args.dir).free, _mem_available()
    if free_disk < 1.1 * computed or free_ram < 1.5 * computed:
        raise SystemExit(f"the state is {computed / 1e9:.1f} GB: {args.dir} has {free_disk / 1e9:.1f} GB free and the "
                         f"host {free_ram / 1e9:.1f} GB of memory available; lower --rollouts")
    for name, n in rows.items():
        buf = getattr(algo, name)
        buf._T = args.T if name == "buffer" else 1
        buf._data = {k: (torch.randint(0, 2, (n, *s), dtype=torch.uint8, device="cuda") if k in ("safe", "unsafe")
                         else torch.rand((n, *s), dtype=torch.float32, device="cuda")) for k, s in shapes.items()}
    torch.cuda.synchronize()
    d = tempfile.mkdtemp(prefix="train_state_", dir=args.dir)
    path = os.path.join(d, "rank0.pt")
    save_s, load_s = [], []
    try:
        for _ in range(args.repeats):
            t0 = time.perf_counter()
            save_train_state(tr, path, 0)
            save_s.append(time.perf_counter() - t0)
            t0 = time.perf_counter()
            load_train_state(tr, path)
            torch.cuda.synchronize()
            load_s.append(time.perf_counter() - t0)
        size = os.path.getsize(path)
    finally:
        shutil.rmtree(d, ignore_errors=True)
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    print(json.dumps({
        "config": cfg["name"], "graphs": rows, "bytes_per_graph": per_graph, "bytes_computed": computed,
        "bytes_file": size, "save_s": [round(s, 3) for s in save_s], "load_s": [round(s, 3) for s in load_s],
        "save_GBps": round(size / min(save_s) / 1e9, 2), "load_GBps": round(size / min(load_s) / 1e9, 2),
        "gpu": q.stdout.strip() if q.returncode == 0 else "unknown", "state_dir_free_GB": round(free_disk / 1e9, 1),
    }), flush=True)


if __name__ == "__main__":
    main()
