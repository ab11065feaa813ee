#!/usr/bin/env python3
"""bench_env_terrain.py -- the cost of per-environment terrain (cassie_batch_set_env_hfield) on a config-4-like workload.

  python tools/bench_env_terrain.py [--steps K] [--warmup W] [--repeats R]

One batch of 4096 fp32 environments on cassie_hfield.xml with a bank of 64 terrains (seeded, as tests/test_env_terrain.py's terrain_bank), the
standing PD rows, settled 600 untimed ticks from the initial drop.  Per arm, timed between CUDA events after W warm-up launches: K single-tick step
launches, K / 50 fifty-tick launches (per tick), K / 10 casts of a 21 x 21 heading-frame height scan and K / 10 renders of a 64 x 64 depth image of the
egocentric camera.  The arms run in turn, R times, each from the same snapshot:
  shared         no terrain rows: environment e on entry e % 64, the shared position and size (the F_ALL / F_EG instances)
  rows_mod_k     selection rows holding e % 64 and the shared position and size: the cost of the F_TR instance alone
  random         random selections, elevation scales U(0, 2) x and position offsets U(-5, 5) cm (seed 4242)
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
    from test_env_terrain import SHARED_POS, SHARED_SIZE, terrain_bank
    P = importlib.import_module('cassie-mujoco-sim_b200')
    n, K = 4096, 64
    torch.cuda.set_device(0)
    b = P.CassieBatch(n, modelfile=P.model_path('cassie_hfield'), precision=P.FP32)
    b.set_stream(torch.cuda.current_stream().cuda_stream)   # the events below are recorded on the stream the batch's launches go to
    b.set_hfield_data(terrain_bank(K, 7) * 0.5)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.set_height_scan(np.linspace(-1.0, 1.0, 21), np.linspace(-1.0, 1.0, 21))
    b.set_camera(name='egocentric', width=64, height=64, zfar=4.0)
    b.step(600)
    snap = b.get_state()
    rng = np.random.default_rng(4242)
    rand = dict(terrain=rng.integers(0, K, n), pos=SHARED_POS + np.c_[rng.uniform(-0.05, 0.05, (n, 3))],
                size=np.c_[np.full(n, SHARED_SIZE[0]), np.full(n, SHARED_SIZE[1]), SHARED_SIZE[2] * rng.uniform(0, 2, n), np.full(n, SHARED_SIZE[3])])

    def timed(fn, count, per=1):
        for _ in range(args.warmup):
            fn()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        e0.record()
        for _ in range(count):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / (count * per)

    K1 = args.steps
    res = {a: {k: [] for k in ('step1_ms', 'step50_ms_per_tick', 'scan_ms', 'depth_ms')} for a in ('shared', 'rows_mod_k', 'random')}
    for _ in range(args.repeats):
        for arm in res:
            b.clear_env_hfield()
            if arm == 'rows_mod_k':
                b.set_env_hfield(terrain=np.arange(n) % K, pos=SHARED_POS, size=SHARED_SIZE)
            elif arm == 'random':
                b.set_env_hfield(**rand)
            b.set_state(snap)
            r = res[arm]
            r['step1_ms'].append(timed(lambda: b.step(1), K1))
            r['step50_ms_per_tick'].append(timed(lambda: b.step(50), max(1, K1 // 50), 50))
            r['scan_ms'].append(timed(b.raycast, max(1, K1 // 10)))
            r['depth_ms'].append(timed(b.render_depth, max(1, K1 // 10)))
    b.clear_env_hfield()
    b.free_state(snap)
    try:
        smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    except OSError:
        smi = ''
    out = {'gpu': smi, 'envs': n, 'terrains': K, 'steps': K1}
    for arm, r in res.items():
        out[arm] = {k: float(np.median(v)) for k, v in r.items()}
    print(json.dumps(out))


if __name__ == '__main__':
    main()
