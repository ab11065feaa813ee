#!/usr/bin/env python3
"""bench_env_contact.py -- the cost of per-environment contact softness (cassie_batch_set_env_contact) on configuration 2's workload.

  python tools/bench_env_contact.py [--steps K] [--warmup W] [--repeats R]

One batch of 4096 fp32 environments of cassie.xml (configuration 2's size) with the standing PD rows, settled 600 untimed ticks.  Per arm, timed
between CUDA events after W warm-up ticks: K single-tick step launches and K / 50 fifty-tick launches (per tick).  The arms run in turn, R times,
each from the same snapshot:
  mechanics_model  mechanics rows holding the model's values (and the actuator, offset and constant rows they bring): the F_MC instance f11c4
  contact_model    contact rows holding the model's values (and the mechanics rows they bring): the F_CT instance f13c4 simulating what f11c4 simulates
  contact          random contact rows (per colliding geom timeconst x U(0.6, 3), dampratio x U(0.5, 1.5), solimp and solmix drawn as
                   tests/contact_support.py random_contact does, seeds 4242 + e): f13c4
Each timed measurement starts from the arm's snapshot, so the single-tick and the 50-tick launches simulate the same ticks.  Prints one JSON line with
the card's name and power limit, the median milliseconds per launch (per tick for the 50-tick launches) and, per arm, the mean constraint rows,
contacts and PGS iterations per environment after the last 50-tick measurement."""
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
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    from contact_support import random_contact
    P = importlib.import_module('cassie-mujoco-sim_b200')
    n = 4096
    torch.cuda.set_device(0)
    parts = ('solref', 'solimp', 'solmix')

    def make(arm):
        b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
        b.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below are recorded on the stream the batch's launches go to
        if arm == 'mechanics_model':
            b.set_env_mechanics(*[v for v in b.env_mechanics().values()])
        elif arm == 'contact_model':
            b.set_env_contact(*[v for v in b.env_contact().values()])
        elif arm == 'contact':
            m = b.env_contact()
            b0 = [m[k][0] for k in parts]
            vals = [random_contact('cassie', 4242 + e, b0) for e in range(n)]
            b.set_env_contact(*[np.stack([v[p] for v in vals]) for p in range(3)])
        b.reset()
        b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        b.step(600)
        return b, b.get_state()

    def timed(b, snap, fn, count, per=1):
        b.set_state(snap)
        for _ in range(max(1, args.warmup // per)):   # the same simulated ticks in both launch shapes: W + K of them
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(count):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (count * per)

    arms = {a: make(a) for a in ('mechanics_model', 'contact_model', 'contact')}
    K1 = args.steps
    res = {a: {k: [] for k in ('step1_ms', 'step50_ms_per_tick')} for a in arms}
    work = {}
    for _ in range(args.repeats):
        for arm, (b, snap) in arms.items():
            res[arm]['step1_ms'].append(timed(b, snap, lambda: b.step(1), K1))
            res[arm]['step50_ms_per_tick'].append(timed(b, snap, lambda: b.step(50), max(1, K1 // 50), 50))
            c = b.counters()
            work[arm] = {'nefc': float(c[:, 0].mean()), 'contacts': float(c[:, 1].mean()), 'pgs_iters': float(c[:, 3].mean())}
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
        out[arm]['per_env_after_last_timed_launch'] = work[arm]
    print(json.dumps(out))


if __name__ == '__main__':
    main()
