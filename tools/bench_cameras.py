"""Cost of camera sets (cassie_batch_set_cameras): 4096 fp32 cassie_depth.xml environments standing on bench.py config 2's motor-PD targets, 64 x 64
pixels, zfar 5.  Three cameras -- the egocentric mount on the pelvis, a camera on the left tarsus looking down, a world-body camera (the rig of
tests/camera_set_support.py) -- rendered in one launch, against the workaround the set replaces: three rounds of set_camera + render_depth + a device
copy of the image.  Then what per-environment mount rows and geom ids add to the three-camera launch, and, with --parent, one camera (the egocentric
one) against another build of the package, in alternating passes in the same process.  Device times from CUDA events over --renders back-to-back
launches after a warm-up, medians of --passes passes.  The GPU's name and power limit are read in the same run.  One JSON line per measurement.

  python tools/bench_cameras.py [--envs 4096] [--renders 200] [--passes 5] [--parent DIR] [--out FILE]

--parent DIR: a directory holding another build of the package (its __init__.py, libcassie_b200.so and models/), imported under its own name."""
import argparse
import importlib
import importlib.util
import json
import os
import statistics
import sys

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, 'tools'), os.path.join(REPO, 'tests'), os.path.join(REPO, 'oracle')]
import bench_raycast as BR  # noqa: E402

SIDE, ZFAR = 64, 5.0


def batch(P, n):
    b = P.CassieBatch(n, modelfile=P.model_path('cassie_depth'), precision=P.FP32)
    b.set_pd(P.pd_rows(n, pTarget=BR.PD_TARGET, pGain=BR.PD_PGAIN, dGain=BR.PD_DGAIN))
    b.step(50)
    return b


def timer(torch, s):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn, reps):
        torch.cuda.synchronize()
        e0.record(s)
        for _ in range(reps):
            fn()
        e1.record(s)
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / reps
    return timed


def rig(b):
    import camera_set_support as CSS
    import test_camera as TC
    q0 = TC.states('cassie_depth', np.random.default_rng(0))[0]
    return CSS.rig('cassie_depth', lambda name: b.name2id('body', name), q0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--envs', type=int, default=4096)
    ap.add_argument('--renders', type=int, default=200)
    ap.add_argument('--passes', type=int, default=5)
    ap.add_argument('--parent', default=None)
    ap.add_argument('--out', default=None)
    args = ap.parse_args()
    import torch
    import camera_set_support as CSS
    P = importlib.import_module('cassie-mujoco-sim_b200')
    P.lib()
    info = BR.gpu_info()
    s = torch.cuda.current_stream()
    timed = timer(torch, s)
    n, R = args.envs, args.renders
    lines = []

    def emit(**kw):
        lines.append(dict(kw, envs=n, width=SIDE, height=SIDE, gpu=info))
        print(json.dumps(lines[-1]), flush=True)

    b = batch(P, n)
    b.set_stream(s.cuda_stream)
    cams = rig(b)
    rows = CSS.random_rows(np.random.default_rng(1), cams, n)

    def set3():
        b.set_cameras(cams, width=SIDE, height=SIDE, zfar=ZFAR)

    def one_launch():
        b.render_depth()
        return b.torch_view('depth').clone()

    def three_rounds():   # the workaround: one camera at a time, each image copied out before the next set drops the rows
        out = []
        for body, pos, quat, fovy in cams:
            b.set_camera(body=b.id2name('body', body), pos=pos, quat=quat, fovy=fovy, width=SIDE, height=SIDE, zfar=ZFAR)
            b.render_depth()
            out.append(b.torch_view('depth').clone())
        return out

    med = {}
    for name, setup, fn in (('three_in_one_launch', set3, one_launch), ('three_set_camera_rounds', None, three_rounds)):
        if setup:
            setup()
        for _ in range(5):
            fn()
        med[name] = statistics.median(timed(fn, max(5, R // 10)) for _ in range(args.passes))
    emit(metric='three_cameras_ms', one_launch_with_copy_ms=med['three_in_one_launch'], three_rounds_ms=med['three_set_camera_rounds'],
         speedup=med['three_set_camera_rounds'] / med['three_in_one_launch'])
    variants = {}
    for name, rows_on, geoms_on in (('plain', False, False), ('rows', True, False), ('geoms', False, True), ('rows_and_geoms', True, True)):
        set3()
        if rows_on:
            b.set_env_cameras(pos=rows[..., 0:3], quat=rows[..., 3:7], fovy=rows[..., 7])
        b.enable_camera_geoms(geoms_on)
        for _ in range(20):
            b.render_depth()
        variants[name] = statistics.median(timed(b.render_depth, R) for _ in range(args.passes))
    b.enable_camera_geoms(False)
    emit(metric='three_camera_render_ms', **{k + '_ms': v for k, v in variants.items()},
         rows_cost=variants['rows'] / variants['plain'] - 1, geoms_cost=variants['geoms'] / variants['plain'] - 1)
    b.close()
    if args.parent:   # one camera, this build against the other, alternating
        d = os.path.abspath(args.parent)
        spec = importlib.util.spec_from_file_location('cassie_other', os.path.join(d, '__init__.py'), submodule_search_locations=[d])
        Q = importlib.util.module_from_spec(spec)
        sys.modules['cassie_other'] = Q
        spec.loader.exec_module(Q)
        builds = []
        for M in (P, Q):
            bb = batch(M, n)
            bb.set_stream(s.cuda_stream)
            bb.set_camera('egocentric', width=SIDE, height=SIDE, zfar=ZFAR)
            for _ in range(20):
                bb.render_depth()
            builds.append(bb)
        times = ([], [])
        for _ in range(args.passes):
            for i, bb in enumerate(builds):
                times[i].append(timed(bb.render_depth, R))
        same = np.array_equal(builds[0].depth(), builds[1].depth())
        emit(metric='one_camera_vs_other_build_ms', this_build_ms=statistics.median(times[0]), other_build_ms=statistics.median(times[1]),
             this_passes=times[0], other_passes=times[1], ratio=statistics.median(times[0]) / statistics.median(times[1]), images_bitwise_equal=bool(same))
        for bb in builds:
            bb.close()
    if args.out:
        with open(args.out, 'w') as f:
            f.write('\n'.join(json.dumps(x) for x in lines) + '\n')


if __name__ == '__main__':
    main()
