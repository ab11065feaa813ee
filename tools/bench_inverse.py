#!/usr/bin/env python3
"""bench_inverse.py -- the cost of the inverse rows (cassie_batch_inverse, launch mode 6) on bench.py's config-2 batch.

  python tools/bench_inverse.py [--launches L] [--repeats R]

One Workload copy of config 2 (4096 envs, fp32, seeded jitter) settles 600 ticks; its acceleration rows' qacc of a forward is copied into the
inverse-input rows on the device.  Then, R times:
  launch_ms          L inverse launches back to back (compute_inverse(None): the input rows as they are) between two CUDA events, divided by L
  launch_and_get_ms  one launch and the synchronous cassie_batch_get_inverse of every part (qfrc_inverse, qfrc_constraint, counts), timed with CUDA
                     events around it (median of 20): what a host consumer of the rows waits for
Prints one JSON line with the medians and the card's name and power limit."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
import bench  # noqa: E402  (Workload, configurations)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--launches', type=int, default=200)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    import torch
    P = importlib.import_module('cassie-mujoco-sim_b200')
    torch.cuda.set_device(0)
    W = bench.Workload(P, 2, bench.CONFIGS[2]['envs'], 0, 0, torch)
    b = W.make_copy(0)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    b.enable_accelerations()
    b.step(600)
    b.forward()
    b.torch_view('inv_qacc')[:, :b.nv].copy_(b.torch_view('acc')[:, P.ACC['qacc']][:, :b.nv])
    b.compute_inverse(None)
    b.sync()
    launch, get = [], []
    for _ in range(args.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.launches):
            b.compute_inverse(None)
        e1.record()
        torch.cuda.synchronize()
        launch.append(e0.elapsed_time(e1) / args.launches)
        t = []
        for _ in range(20):
            e0.record()
            b.compute_inverse(None)
            b.inverse()
            e1.record()
            torch.cuda.synchronize()
            t.append(e0.elapsed_time(e1))
        get.append(float(np.median(t)))
    props = torch.cuda.get_device_properties(0)
    try:
        pl = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'], capture_output=True, text=True).stdout.strip()
        power = float(pl.splitlines()[0]) if pl else None
    except Exception:
        power = None
    print(json.dumps({'metric': 'Cassie inverse rows, config 2 batch', 'envs': W.n, 'launches': args.launches,
                      'device': {'name': props.name, 'sms': props.multi_processor_count, 'power_limit_w': power},
                      'launch_ms': launch, 'launch_ms_median': float(np.median(launch)), 'launch_and_get_ms': get, 'launch_and_get_ms_median': float(np.median(get))}), flush=True)
    b.close()


if __name__ == '__main__':
    main()
