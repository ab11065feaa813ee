#!/usr/bin/env python3
"""bench_trace.py -- the cost of per-tick traces (cassie_batch_set_trace) on a 40 Hz policy step of a 2 kHz simulation: 50 ticks per policy step.

  python tools/bench_trace.py [--steps K] [--warmup W] [--repeats R]

One batch of 4096 fp32 environments of cassie.xml per arm, derived-quantity rows on, the standing PD rows, settled 600 untimed ticks.  Per arm, K policy
steps timed between CUDA events after W warm-up policy steps, each arm from the same snapshot, the arms in turn, R times:
  chain       one 50-tick launch on the applied-force chain twin (zeroed applied rows), no trace: f17c4
  traced      one 50-tick launch with a 16-column trace -- the z foot forces, the foot heights, the pelvis height, the ten motor torques and the pelvis
              forward velocity -- on its F_TC twin: f1fc4
  single      today's workaround: 50 single-tick launches (f14), the same 16 columns gathered after each from torch_view('aux' / 'qpos' / 'qvel' /
              'obs') into a [n, 50, 16] tensor on the batch's stream
Prints one JSON line with the card's name and power limit, the median milliseconds per policy step and the env-steps (ticks) per second."""
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
    ap.add_argument('--steps', type=int, default=40)
    ap.add_argument('--warmup', type=int, default=4)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    import torch
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    P = importlib.import_module('cassie-mujoco-sim_b200')
    n, ticks = 4096, 50
    torch.cuda.set_device(0)
    cols = [(P.TRACE_AUX, 2), (P.TRACE_AUX, 8), (P.TRACE_AUX, 26), (P.TRACE_AUX, 29), (P.TRACE_QPOS, 2)] + \
        [(P.TRACE_OBS, c) for c in range(20, 30)] + [(P.TRACE_QVEL, 0)]

    def make(arm):
        b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
        b.set_stream(torch.cuda.current_stream().cuda_stream)   # the events and the gathers below are on the stream the launches go to
        b.enable_aux()
        if arm == 'chain':
            b.enable_applied_forces()
        if arm == 'traced':
            b.set_trace(cols, ticks)
        b.reset()
        b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        b.step(600)
        return b, b.get_state()

    def stepper(arm, b):
        if arm != 'single':
            return lambda: b.step(ticks)
        views = {P.TRACE_AUX: b.torch_view('aux'), P.TRACE_QPOS: b.torch_view('qpos'), P.TRACE_QVEL: b.torch_view('qvel'), P.TRACE_OBS: b.torch_view('obs')}
        out = torch.empty((n, ticks, len(cols)), dtype=torch.float32, device='cuda')
        srcs = [(views[s], c) for s, c in cols]

        def fn():
            for t in range(ticks):
                b.step(1)
                out[:, t] = torch.stack([v[:, c] for v, c in srcs], dim=1)
        return fn

    def timed(b, snap, arm):
        b.set_state(snap)
        fn = stepper(arm, b)
        for _ in range(args.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(args.steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / args.steps

    names = ('chain', 'traced', 'single')
    arms = {a: make(a) for a in names}
    res = {a: [] for a in names}
    for _ in range(args.repeats):
        for arm, (b, snap) in arms.items():
            res[arm].append(timed(b, snap, arm))
    for b, snap in arms.values():
        b.free_state(snap)
        b.close()
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = ''
    out = {'gpu': smi, 'envs': n, 'ticks_per_policy_step': ticks, 'policy_steps': args.steps, 'repeats': args.repeats, 'columns': len(cols)}
    for arm, r in res.items():
        ms = float(np.median(r))
        out[arm] = {'ms_per_policy_step': ms, 'M_env_steps_per_s': n * ticks / ms / 1e3, 'all_ms': [round(x, 4) for x in r]}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
