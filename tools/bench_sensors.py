#!/usr/bin/env python3
"""bench_sensors.py -- the cost of sensor models (cassie_batch_set_env_sensors) on configuration 2's workload.

  python tools/bench_sensors.py [--steps K] [--warmup W] [--repeats R]

One batch of 4096 fp32 environments of cassie.xml per arm, with the standing PD rows, settled 600 untimed ticks.  Per arm, timed between CUDA events
after W warm-up ticks: K single-tick step launches and K / 50 fifty-tick launches (per tick).  The arms run in turn, R times, each from the same snapshot:
  f04            no rows
  f0404          zeroed applied-force rows: the plain twin f0404
  f02404_zero    the zero sensor model: f02404
  f02404_noisy   the model files' noise (shin / tarsus encoders 2e-4, gyro 5e-4, accelerometer 1e-2) on every encoder and IMU channel, offsets, a
                 tilted mount and biases: f02404
  f17c4          contact rows holding the model's values and zeroed applied-force rows: the chain twin f17c4
  f127c4         the same with the noisy sensor model: f127c4
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
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    P = importlib.import_module('cassie-mujoco-sim_b200')
    n = 4096
    torch.cuda.set_device(0)
    rng = np.random.default_rng(0)
    noisy = dict(enc_offset=rng.uniform(-1e-3, 1e-3, (n, 16)), enc_noise=np.full(16, 2e-4), imu_quat=[1.0, 0.01, -0.01, 0.005],
                 imu_bias=rng.uniform(-0.01, 0.01, (n, 6)), imu_noise=[1e-3] * 3 + [5e-4] * 3 + [1e-2] * 3)

    def make(arm):
        b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
        b.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below are recorded on the stream the batch's launches go to
        if arm in ('f17c4', 'f127c4'):
            b.set_env_contact(*[v for v in b.env_contact().values()])
        if arm in ('f0404', 'f17c4'):
            b.enable_applied_forces()
        if arm == 'f02404_zero':
            b.set_env_sensors(imu_quat=[1.0, 0, 0, 0])
        if arm in ('f02404_noisy', 'f127c4'):
            b.set_env_sensors(**noisy)
        b.reset()
        b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        b.step(600)
        return b, b.get_state()

    def timed(b, snap, count, per=1):
        b.set_state(snap)
        for _ in range(max(1, args.warmup // per)):   # the same simulated ticks in both launch shapes: W + K of them
            b.step(per)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(count):
            b.step(per)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (count * per)

    names = ('f04', 'f0404', 'f02404_zero', 'f02404_noisy', 'f17c4', 'f127c4')
    arms = {a: make(a) for a in names}
    K1 = args.steps
    res = {a: {k: [] for k in ('step1_ms', 'step50_ms_per_tick')} for a in arms}
    for _ in range(args.repeats):
        for arm, (b, snap) in arms.items():
            res[arm]['step1_ms'].append(timed(b, snap, K1))
            res[arm]['step50_ms_per_tick'].append(timed(b, snap, max(1, K1 // 50), 50))
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
        out[arm]['spread'] = {k: [float(min(v)), float(max(v))] for k, v in r.items()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
