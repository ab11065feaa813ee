#!/usr/bin/env python3
"""bench_env_geoms.py -- the cost of per-environment static-geom rows (cassie_batch_set_env_geom_pose) on bench.py's config-2 workload.

  python tools/bench_env_geoms.py [--steps K] [--warmup W] [--repeats R]

Each arm is timed like bench.py's `value`: the same Workload copies (4096 envs each, seeded jitter, > 1.5 x L2 in all, stepped round-robin),
exactly K single-tick launches in up to 5 blocks between CUDA events, the median block's time per step.  Before an arm every copy settles 600
untimed ticks and W warm-up ticks; afterwards its rows are dropped and its state is restored from a snapshot.  The arms run in turn, R times:
  shared              no rows: the shipped instances (bench.py's value)
  per_env_geoms_flat  rows holding the model's own placement: the cost of reading the rows
  per_env_stairs      a seeded layout per environment (seed 4242 + 1000 copy): box1 under the left foot and box7 under the right (half-sizes
                      .25 .1 .1, tops at U(0, 5 cm), yaw U(-0.2, 0.2) rad each) and the floor tilted about x by U(-3, 3) degrees; environments on
                      boxes run the box narrow phase and the second collision run
dropped_contacts: contacts beyond 12 per environment in the timed window.  Prints one JSON line with the card's name and power limit."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402  (Workload, L2 size, block count)


def layout(b, j):
    n = b.n
    rng = np.random.default_rng(4242 + 1000 * j)
    for name, y in (('box1', 0.135), ('box7', -0.135)):
        h, yaw = rng.uniform(0.0, 0.05, n), rng.uniform(-0.2, 0.2, n)
        pos = np.stack([np.full(n, 0.05), np.full(n, y), h - 0.1], 1)
        quat = np.stack([np.cos(yaw / 2), np.zeros(n), np.zeros(n), np.sin(yaw / 2)], 1)
        b.set_env_geom_pose(name, pos=pos, quat=quat, size=[0.25, 0.1, 0.1])
    tilt = np.deg2rad(rng.uniform(-3.0, 3.0, n))
    b.set_env_geom_pose('floor', quat=np.stack([np.cos(tilt / 2), np.sin(tilt / 2), np.zeros(n), np.zeros(n)], 1))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=500)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    import torch
    P = importlib.import_module('cassie-mujoco-sim_b200')
    torch.cuda.set_device(0)
    W = bench.Workload(P, 2, bench.CONFIGS[2]['envs'], 0, 0, torch)
    b0 = W.make_copy(0)
    nb = max(2, -(-int(1.5 * bench.L2_BYTES) // W.footprint(b0)))
    copies = [b0] + [W.make_copy(k) for k in range(1, nb)]
    K = args.steps

    def run_arm(arm):
        snaps = [bk.get_state() for bk in copies]
        for j, bk in enumerate(copies):
            if arm == 'per_env_geoms_flat':
                bk.set_env_geom_pose('floor')          # rows holding the model's placement
            elif arm == 'per_env_stairs':
                layout(bk, j)
        for bk in copies:
            bk.step(600)
        for _ in range(args.warmup):
            for bk in copies:
                bk.step(1)
        d0 = sum(int(bk.counters()[:, 4].sum()) for bk in copies)
        sizes = [len(a) for a in np.array_split(np.arange(K), min(bench.MAX_BLOCKS, K))]
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in sizes]
        torch.cuda.synchronize()
        i = 0
        for (e0, e1), m in zip(ev, sizes):
            e0.record()
            for _ in range(m):
                copies[i % nb].step(1); i += 1
            e1.record()
        torch.cuda.synchronize()
        per = [e0.elapsed_time(e1) / m for (e0, e1), m in zip(ev, sizes)]
        dropped = sum(int(bk.counters()[:, 4].sum()) for bk in copies) - d0
        for bk, sn in zip(copies, snaps):
            bk.clear_env_geom_poses(); bk.set_state(sn); bk.free_state(sn)
        ms = float(np.median(per))
        return {'env_steps_per_s': W.n / (ms * 1e-3), 'ms_per_step': ms, 'spread': (max(per) - min(per)) / ms, 'dropped_contacts': dropped}

    arms = ('shared', 'per_env_geoms_flat', 'per_env_stairs')
    runs = {a: [] for a in arms}
    for _ in range(args.repeats):
        for a in arms:
            runs[a].append(run_arm(a))
    props = torch.cuda.get_device_properties(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True).stdout.strip()
        power = float(pl.splitlines()[0]) if pl else None
    except Exception:
        power = None
    print(json.dumps({'metric': 'Cassie env-steps/s, config 2, per-environment static geoms', 'steps': K, 'warmup': args.warmup, 'copies': nb,
                      'device': {'name': props.name, 'sms': props.multi_processor_count, 'power_limit_w': power}, 'runs': runs}), flush=True)
    for bk in copies:
        bk.close()


if __name__ == '__main__':
    main()
