"""Cost of a terrain ray cast (cassie_batch_raycast) on bench.py's config-2 batch: 4096 fp32 environments standing on motor-PD targets, the 17 x 11
heading-frame height scan at 0.1 m (187 rays), on three terrains: the flat floor, per-environment stairs and floor tilt, and config 4's bank of 64
height fields.  Prints one JSON line per terrain with the device time of one raycast launch (CUDA events over --casts back-to-back launches, after a
warm-up), of a launch plus get_rays (host clock, synchronous), and of one single-tick step launch of the same batch for scale.  The GPU's name and
power limit are read in the same run.

  python tools/bench_raycast.py [--envs 4096] [--casts 500] [--out FILE]"""
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
PD_TARGET = [0.0045, 0, 0.4973, -1.1997, -1.5968, -0.0045, 0, 0.4973, -1.1997, -1.5968]
PD_PGAIN, PD_DGAIN = [70, 70, 100, 100, 50] * 2, [7, 7, 8, 8, 5] * 2


def gpu_info():
    try:
        return subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'], text=True).strip()
    except Exception as ex:
        return 'unknown (%r)' % ex


def make(P, terrain, n):
    name = 'cassie_hfield' if terrain == 'bank' else 'cassie'
    b = P.CassieBatch(n, modelfile=P.model_path(name), precision=P.FP32)
    if terrain == 'bank':
        t = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
        t[:, 95:105, 95:105] = 0
        b.set_hfield_data(t)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    if terrain == 'stairs':
        rng = np.random.default_rng(3)
        for j in range(6):
            yaw = rng.uniform(-np.pi, np.pi, n)
            b.set_env_geom_pose(_box_name(P, j), pos=np.column_stack([rng.uniform(-1, 1, n), rng.uniform(-0.7, 0.7, n), rng.uniform(-0.1, 0.1, n)]),
                                quat=np.stack([np.cos(yaw / 2), 0 * yaw, 0 * yaw, np.sin(yaw / 2)], 1), size=rng.uniform([0.1, 0.1, 0.05], [0.5, 0.5, 0.2], (n, 3)))
        tilt = rng.uniform(0, 0.1, n)
        b.set_env_geom_pose('floor', quat=np.stack([np.cos(tilt / 2), np.sin(tilt / 2), 0 * tilt, 0 * tilt], 1))
    b.step(50)
    b.set_height_scan(np.arange(-8, 9) * 0.1, np.arange(-5, 6) * 0.1)
    return b


def _box_name(P, j):
    """the j-th box geom of the world body in cassie.xml (the stair boxes)"""
    t = {ln.split()[0]: ln.split()[3:] for ln in open(P.model_path('cassie')) if not ln.startswith('#')}
    names, types, bodies = t['names_geom'], [int(x) for x in t['geom_type']], [int(x) for x in t['geom_bodyid']]
    return [nm for nm, t, bd in zip(names, types, bodies) if t == 6 and bd == 0][j]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--casts', type=int, default=500)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    P = importlib.import_module('cassie-mujoco-sim_b200')
    P.lib()
    info = gpu_info()
    lines = []
    for terrain in ('flat', 'stairs', 'bank'):
        b = make(P, terrain, args.envs)
        s = torch.cuda.current_stream()
        b.set_stream(s.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        for _ in range(50):
            b.raycast()
            b.step(1)
        torch.cuda.synchronize()
        e0.record(s)
        for _ in range(args.casts):
            b.raycast()
        e1.record(s)
        torch.cuda.synchronize()
        cast_ms = e0.elapsed_time(e1) / args.casts
        e0.record(s)
        for _ in range(args.casts):
            b.step(1)
        e1.record(s)
        torch.cuda.synchronize()
        step_ms = e0.elapsed_time(e1) / args.casts
        t0 = time.perf_counter()
        for _ in range(50):
            b.raycast()
            b.rays()
        get_ms = (time.perf_counter() - t0) / 50 * 1e3
        r = b.rays()
        lines.append(dict(metric='raycast_ms', terrain=terrain, envs=args.envs, rays=b.nrays(), cast_ms=cast_ms, cast_plus_get_rays_ms=get_ms, step_1tick_ms=step_ms,
                          cast_over_step=cast_ms / step_ms, rays_per_s=args.envs * b.nrays() / (cast_ms * 1e-3), hit_fraction=float((r[:, :, 0] >= 0).mean()), gpu=info))
        print(json.dumps(lines[-1]))
        b.close()
    if args.out:
        with open(args.out, 'w') as f:
            f.write('\n'.join(json.dumps(x) for x in lines) + '\n')


if __name__ == '__main__':
    main()
