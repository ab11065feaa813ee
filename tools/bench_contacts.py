#!/usr/bin/env python3
"""bench_contacts.py -- the cost of contact lists (cassie_batch_enable_contacts) on the launches that carry them.

  python tools/bench_contacts.py [--steps K] [--warmup W] [--repeats R]

Two batches of 4096 fp32 environments of cassie.xml (config 2: the standing PD rows), acceleration rows on, settled 600 untimed ticks:
  chain     model-valued applied rows: the F_FR chain twin f17d7
  listed    contact lists: its F_CL twin f117d7
Per arm and launch length (1 tick, 50 ticks), K launches timed between CUDA events after W warm-up launches, the arms alternated, R times.  Prints one
JSON line with the card's name and power limit and the median milliseconds per launch."""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tests'))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--steps', type=int, default=200)
    ap.add_argument('--warmup', type=int, default=20)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    import torch
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    P = importlib.import_module('cassie-mujoco-sim_b200')
    n = 4096
    torch.cuda.set_device(0)
    arms = {}
    for name in ('chain', 'listed'):
        b = P.CassieBatch(n, precision=P.FP32)
        b.enable_accelerations()
        if name == 'chain':
            b.enable_applied_forces()
        else:
            b.enable_contacts()
        b.set_pd(P.pd_rows(n, pTarget=np.tile(PD_TARGET, (n, 1)), pGain=PD_PGAIN, dGain=PD_DGAIN))
        b.step(600)
        b.sync()
        arms[name] = b
    times = {(a, t): [] for a in arms for t in (1, 50)}
    for _ in range(args.repeats):
        for ticks in (1, 50):
            steps = args.steps if ticks == 1 else max(1, args.steps // 10)
            for a, b in arms.items():
                for _ in range(args.warmup):
                    b.step(ticks)
                b.sync()
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                for _ in range(steps):
                    b.step(ticks)
                b.sync()
                e.record()
                e.synchronize()
                times[(a, ticks)].append(s.elapsed_time(e) / steps)
    gpu = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    out = dict(gpu=gpu, envs=n, model='cassie.xml', precision='fp32')
    for (a, t), v in times.items():
        ms = float(np.median(v))
        out['%s_%dtick_ms' % (a, t)] = ms
        out['%s_%dtick_env_steps_per_s' % (a, t)] = n * t / ms * 1e3
    for t in (1, 50):
        out['listed_over_chain_%dtick' % t] = out['listed_%dtick_ms' % t] / out['chain_%dtick_ms' % t] - 1
    print(json.dumps(out))
    for b in arms.values():
        b.close()


if __name__ == '__main__':
    main()
