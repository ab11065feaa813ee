"""Cost of a depth render (cassie_batch_render_depth) on bench.py's config-2 batch: 4096 fp32 environments standing on motor-PD targets, with the
egocentric camera of cassie_depth.xml (on the pelvis, 0.2 m ahead and above, looking 45 degrees down, fovy 65.5), at 32 x 32 and 64 x 64 pixels, on
three scenes: the flat floor, per-environment stairs, and config 4's bank of 64 height fields.  Prints one JSON line per scene and size with the device
time of one render launch (CUDA events over --renders back-to-back launches, after a warm-up), Mpixel/s, the time of a single-tick step launch and of
a 50-tick step launch of the same batch, and whether a render every 50 ticks (a 40 Hz policy) costs less than those 50 ticks.  The GPU's name and
power limit are read in the same run.

  python tools/bench_camera.py [--envs 4096] [--renders 200] [--out FILE]"""
import argparse
import importlib
import json
import os
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, 'tools'))
import bench_raycast as BR  # noqa: E402


def egocentric(P):
    """the egocentric camera of cassie_depth.xml (pose in the pelvis frame, fovy), from the compiled table"""
    t = {ln.split()[0]: ln.split()[3:] for ln in open(P.model_path('cassie_depth')) if not ln.startswith('#')}
    k = t['names_camera'].index('egocentric')
    return [float(x) for x in t['camera_pos'][3 * k:3 * k + 3]], [float(x) for x in t['camera_quat'][4 * k:4 * k + 4]], float(t['camera_fovy'][k])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--renders', type=int, default=200)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    P = importlib.import_module('cassie-mujoco-sim_b200')
    P.lib()
    info = BR.gpu_info()
    pos, quat, fovy = egocentric(P)
    lines = []
    for scene in ('flat', 'stairs', 'bank'):
        b = BR.make(P, scene, args.envs)   # the ray benchmark's batches: same terrains, 50 settling ticks
        s = torch.cuda.current_stream()
        b.set_stream(s.cuda_stream)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

        def timed(fn, reps):
            torch.cuda.synchronize()
            e0.record(s)
            for _ in range(reps):
                fn()
            e1.record(s)
            torch.cuda.synchronize()
            return e0.elapsed_time(e1) / reps

        for _ in range(20):
            b.step(1)
        step1 = timed(lambda: b.step(1), args.renders)
        step50 = timed(lambda: b.step(50), max(5, args.renders // 20))
        for side in (32, 64):
            b.set_camera(body='cassie-pelvis', pos=pos, quat=quat, fovy=fovy, width=side, height=side, zfar=5.0)
            for _ in range(20):
                b.render_depth()
            ms = timed(b.render_depth, args.renders)
            d = b.depth()
            lines.append(dict(metric='render_depth_ms', scene=scene, envs=args.envs, width=side, height=side, render_ms=ms,
                              mpixel_per_s=args.envs * side * side / (ms * 1e-3) / 1e6, step_1tick_ms=step1, render_over_step_1tick=ms / step1,
                              step_50tick_ms=step50, render_every_50_ticks_cheaper=bool(ms < step50), hit_fraction=float((d < 5.0).mean()), gpu=info))
            print(json.dumps(lines[-1]))
        b.close()
    if args.out:
        with open(args.out, 'w') as f:
            f.write('\n'.join(json.dumps(x) for x in lines) + '\n')


if __name__ == '__main__':
    main()
