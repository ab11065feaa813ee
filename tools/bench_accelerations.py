#!/usr/bin/env python3
"""bench_accelerations.py -- the cost of acceleration rows (cassie_batch_enable_accelerations) on bench.py's config-2 workload.

  python tools/bench_accelerations.py [--steps K] [--warmup W] [--repeats R]

Each arm is timed like bench.py's `value`: the same Workload copies (4096 fp32 envs each, seeded jitter, > 1.5 x L2 in all, stepped round-robin),
exactly K single-tick launches in up to 5 blocks between CUDA events, the median block's time per step.  Before an arm every copy settles 600
untimed ticks and W warm-up ticks; afterwards its rows are dropped and its state is restored from a snapshot.  The arms run in turn, R times:
  frames_8      8 frames (cassie-pelvis, left-foot, right-foot, the four toe / heel sites and imu) without acceleration rows: the extended F_FR instance
  frames_8_acc  the same 8 frames with acceleration rows (qacc and the cacc of the 8 frames)
  acc_only      acceleration rows without frames (qacc only), on the same F_FR instance
Prints one JSON line with the card's name and power limit."""
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

EIGHT = (['cassie-pelvis', 'left-foot', 'right-foot', 'left-toe', 'left-heel', 'right-toe', 'right-heel', 'imu'], [0, 0, 0, 1, 1, 1, 1, 1])


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
    arms = {'frames_8': (EIGHT, False), 'frames_8_acc': (EIGHT, True), 'acc_only': (None, True)}

    def run_arm(arm):
        frames, acc = arms[arm]
        snaps = [bk.get_state() for bk in copies]
        for bk in copies:
            if frames:
                bk.set_frames(*frames)
            bk.enable_accelerations(acc)
        for bk in copies:
            bk.step(600)
        for _ in range(args.warmup):
            for bk in copies:
                bk.step(1)
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
        for bk, sn in zip(copies, snaps):
            bk.set_frames([]); bk.enable_accelerations(False); bk.set_state(sn); bk.free_state(sn)
        ms = float(np.median(per))
        return {'env_steps_per_s': W.n / (ms * 1e-3), 'ms_per_step': ms, 'spread': (max(per) - min(per)) / ms}

    runs = {a: [] for a in arms}
    for _ in range(args.repeats):
        for a in arms:
            runs[a].append(run_arm(a))
    med = {a: float(np.median([r['env_steps_per_s'] for r in runs[a]])) for a in arms}
    props = torch.cuda.get_device_properties(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True).stdout.strip()
        power = float(pl.splitlines()[0]) if pl else None
    except Exception:
        power = None
    print(json.dumps({'metric': 'Cassie env-steps/s, config 2, acceleration rows', 'steps': K, 'warmup': args.warmup, 'copies': nb,
                      'device': {'name': props.name, 'sms': props.multi_processor_count, 'power_limit_w': power}, 'runs': runs, 'median': med,
                      'acc_cost_vs_frames_8': 1 - med['frames_8_acc'] / med['frames_8']}), flush=True)
    for bk in copies:
        bk.close()


if __name__ == '__main__':
    main()
