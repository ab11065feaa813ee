#!/usr/bin/env python3
"""bench_frames.py -- the cost of frame rows (cassie_batch_set_frames) on bench.py's config-2 workload.

  python tools/bench_frames.py [--steps K] [--warmup W] [--repeats R]

Each arm is timed like bench.py's `value`: the same Workload copies (4096 envs each, seeded jitter, > 1.5 x L2 in all, stepped round-robin),
exactly K single-tick launches in up to 5 blocks between CUDA events, the median block's time per step.  Before an arm every copy settles 600
untimed ticks and W warm-up ticks; afterwards its frames are dropped and its state is restored from a snapshot.  The arms run in turn, R times:
  no_frames   the shipped plain instance (bench.py's value)
  aux_only    the shipped extended instance with aux rows and no frames: what the switch to the extended instance costs by itself
  frames_8    cassie-pelvis, left-foot, right-foot, the four toe / heel sites and imu: the extended F_FR instance
  frames_all  every body and every site of cassie.xml (39 frames: two lane passes per stage)
Then the time of one frame_jacobian call (one mode-4 launch and the host copy) on one copy of 4096 envs, median of 20.  Prints one JSON line with the card's name and power limit."""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402  (Workload, L2 size, block count)

EIGHT = (['cassie-pelvis', 'left-foot', 'right-foot', 'left-toe', 'left-heel', 'right-toe', 'right-heel', 'imu'], [0, 0, 0, 1, 1, 1, 1, 1])


def model_frames():
    """every body and site named in cassie.xml's model table"""
    names = {}
    with open(os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models', 'cassie.cmodel')) as f:
        for ln in f:
            t = ln.split()
            if t and t[0] in ('names_body', 'names_site'):
                names[t[0]] = t[3:]
    return names['names_body'] + names['names_site'], [0] * len(names['names_body']) + [1] * len(names['names_site'])


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
    arms = {'no_frames': None, 'aux_only': None, 'frames_8': EIGHT, 'frames_all': model_frames()}

    def run_arm(arm):
        snaps = [bk.get_state() for bk in copies]
        for bk in copies:
            if arms[arm]:
                bk.set_frames(*arms[arm])
            elif arm == 'aux_only':
                bk.enable_aux(True)
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
            bk.set_frames([]); bk.enable_aux(False); bk.set_state(sn); bk.free_state(sn)
        ms = float(np.median(per))
        return {'env_steps_per_s': W.n / (ms * 1e-3), 'ms_per_step': ms, 'spread': (max(per) - min(per)) / ms}

    runs = {a: [] for a in arms}
    for _ in range(args.repeats):
        for a in arms:
            runs[a].append(run_arm(a))
    # what reading the rows back costs: a synchronous host copy of every frame row of one copy (4096 envs x 39 frames)
    copies[0].set_frames(*arms['frames_all'])
    copies[0].step(1)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(20):
        copies[0].frames()
    get_ms = (time.perf_counter() - t0) / 20 * 1e3
    jac_ms = []
    for _ in range(21):
        t0 = time.perf_counter()
        copies[0].frame_jacobian(2)
        jac_ms.append((time.perf_counter() - t0) * 1e3)
    jac_ms = float(np.median(jac_ms[1:]))
    copies[0].set_frames([])
    props = torch.cuda.get_device_properties(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True).stdout.strip()
        power = float(pl.splitlines()[0]) if pl else None
    except Exception:
        power = None
    print(json.dumps({'metric': 'Cassie env-steps/s, config 2, frame rows', 'steps': K, 'warmup': args.warmup, 'copies': nb,
                      'device': {'name': props.name, 'sms': props.multi_processor_count, 'power_limit_w': power}, 'runs': runs,
                      'frames_all_host_copy_ms': get_ms, 'frame_jacobian_ms': jac_ms}), flush=True)
    for bk in copies:
        bk.close()


if __name__ == '__main__':
    main()
