#!/usr/bin/env python3
"""bench_applied_forces.py -- the cost of per-environment applied forces (cassie_batch_set_applied_forces) on configuration 2 / 3's workload.

  python tools/bench_applied_forces.py [--steps K] [--warmup W] [--repeats R]

One batch of 4096 fp32 environments of cassie.xml per arm, with the standing PD rows, settled 600 untimed ticks.  Per arm, timed between CUDA events
after W warm-up ticks: K single-tick step launches and K / 50 fifty-tick launches (per tick).  The arms run in turn, R times, each from the same snapshot:
  plain          no rows: f04
  plain_zero     zeroed applied-force rows: the plain twin f0404
  contact_model  contact rows holding the model's values: f13c4
  chain_zero     the same plus zeroed applied-force rows: the chain twin f17c4
  push_device    configuration 3's push schedule (Philox seed 1234 keyed by environment and event, xy ~ U(-100, 100) N on the pelvis, held 100 ticks of
                 every 400) written into torch_view('applied') between launches: f0404
  push_slot      the same schedule through cassie_batch_apply_force / clear_forces, each a synchronous upload: f04
Prints one JSON line with the card's name and power limit and the median milliseconds per launch (per tick for the 50-tick launches)."""
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
    ap.add_argument('--steps', type=int, default=500)
    ap.add_argument('--warmup', type=int, default=50)
    ap.add_argument('--repeats', type=int, default=3)
    args = ap.parse_args()
    import torch
    import bench
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    P = importlib.import_module('cassie-mujoco-sim_b200')
    n = 4096
    torch.cuda.set_device(0)
    pushes = [torch.as_tensor(bench.philox_uniform(1234, k, (n, 2), -100.0, 100.0), dtype=torch.float32, device='cuda') for k in range(8)]
    pushes_host = [bench.philox_uniform(1234, k, (n, 2), -100.0, 100.0) for k in range(8)]

    def make(arm):
        b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
        b.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below are recorded on the stream the batch's launches go to
        if arm in ('contact_model', 'chain_zero'):
            b.set_env_contact(*[v for v in b.env_contact().values()])
        if arm in ('plain_zero', 'chain_zero', 'push_device'):
            b.enable_applied_forces()
        b.reset()
        b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        b.step(600)
        return b, b.get_state()

    def stepper(arm, b):
        """fn(ticks): one launch of `ticks` ticks, with the arm's push schedule applied at its tick boundaries"""
        clock = [0]
        view = b.torch_view('applied') if arm == 'push_device' else None

        def fn(ticks):
            t = clock[0]
            if arm == 'push_device':
                if t % 400 == 0:
                    view[:, 6:8] = pushes[(t // 400) % 8]
                elif t % 400 == 100:
                    view[:, 6:8] = 0
            elif arm == 'push_slot':
                if t % 400 == 0:
                    push = np.zeros((n, 6))
                    push[:, :2] = pushes_host[(t // 400) % 8]
                    b.apply_force(push, 'cassie-pelvis')
                elif t % 400 == 100:
                    b.clear_forces()
            b.step(ticks)
            clock[0] = t + ticks
        return fn, clock

    def timed(b, snap, arm, count, per=1):
        b.set_state(snap)
        fn, clock = stepper(arm, b)
        for _ in range(max(1, args.warmup // per)):   # the same simulated ticks in both launch shapes: W + K of them
            fn(per)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(count):
            fn(per)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (count * per)

    names = ('plain', 'plain_zero', 'contact_model', 'chain_zero', 'push_device', 'push_slot')
    arms = {a: make(a) for a in names}
    K1 = args.steps
    res = {a: {k: [] for k in ('step1_ms', 'step50_ms_per_tick')} for a in arms}
    for _ in range(args.repeats):
        for arm, (b, snap) in arms.items():
            res[arm]['step1_ms'].append(timed(b, snap, arm, K1))
            res[arm]['step50_ms_per_tick'].append(timed(b, snap, arm, max(1, K1 // 50), 50))
    for b, snap in arms.values():
        b.free_state(snap)
        b.close()
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = ''
    out = {'gpu': smi, 'envs': n, 'steps': K1, 'repeats': args.repeats}
    for arm, r in res.items():
        out[arm] = {k: float(np.median(v)) for k, v in r.items()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
