#!/usr/bin/env python3
"""bench_stages.py -- where the step kernel's time goes: SM clock cycles per stage of a physics sub-step, read from a stage-clock build.

  python tools/bench_stages.py --build DIR                   compile the library with -DCASSIE_STAGE_CLOCKS into DIR (objects in DIR/_obj): no GPU needed
  python tools/bench_stages.py --lib DIR/libcassie_b200.so [--ticks T] [--envs N]

A stage-clock build is the shipped source with lane 0 of every warp recording clock64() at the stage boundaries of mj_substep (csrc/step_core.inl
STAGE_CLOCK) into its environment's qM scratch row; the shipped library never carries it.  The run steps N fp32 environments of cassie.xml under
configuration 2's controller (the standing motor-PD rows of bench.py), settled 600 ticks, then T single-tick launches; after each launch every
environment's stage clocks are read.  Reported per stage: the median over environments and launches of its cycles, and its share of the median
sub-step.  The clocks are per SM, so a stage's figure includes the cycles other warps on its SM took from it: it is the time a warp spends there at
the launch's occupancy, not an instruction count.  Prints one JSON line with the card's name and power limit."""
import argparse
import importlib.util
import json
import os
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PKG = os.path.join(REPO, 'cassie-mujoco-sim_b200')
sys.path.insert(0, os.path.join(REPO, 'tests'))
# STAGE_CLOCK(i) marks in mj_substep; stage k runs from mark k to mark k + 1
STAGES = ['kinematics_compos', 'crb', 'factor_ld', 'velocity_smooth', 'sensors_pos_vel', 'collision', 'constraint_rows', 'constraint_solve',
          'contact_forces_accel', 'euler_solve_m', 'integrate']
NM_MAX = 320


def build(out):
    extra = os.environ.get('CASSIE_B200_NVCC_EXTRA', '').split()
    os.environ['CASSIE_B200_NVCC_EXTRA'] = ' '.join(extra + ([] if '-DCASSIE_STAGE_CLOCKS' in extra else ['-DCASSIE_STAGE_CLOCKS']))
    spec = importlib.util.spec_from_file_location('_cassie_b200_build_stages', os.path.join(PKG, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    out = os.path.abspath(out)
    mod.OBJ = os.path.join(out, '_obj')   # never the shipped objects and resource reports
    os.makedirs(out, exist_ok=True)
    return mod.build(force=True, out=os.path.join(out, 'libcassie_b200.so'))


def run(lib, ticks, n):
    import numpy as np
    import torch
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    spec = importlib.util.spec_from_file_location('cassie_b200_stages', os.path.join(PKG, '__init__.py'), submodule_search_locations=[PKG])
    P = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(P)
    P.LIB_PATH = os.path.abspath(lib)
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    torch.cuda.set_device(0)
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    ptr = b.device_ptr('stage_clocks')
    if not ptr:
        raise SystemExit('%s is not a stage-clock build (python tools/bench_stages.py --build DIR)' % lib)

    class _Arr:
        pass
    a = _Arr()
    a.__cuda_array_interface__ = dict(shape=(n, 2 * NM_MAX), typestr='<u4', data=(ptr, False), version=2)
    rows = torch.as_tensor(a, device='cuda')
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.reset()
    b.step(600)
    b.sync()
    samples = []
    for _ in range(ticks):
        b.step(1)
        b.sync()
        samples.append(rows[:, :len(STAGES) + 1].cpu().numpy().astype(np.int64))
    c = np.concatenate(samples)
    d = (c[:, 1:] - c[:, :-1]) % (1 << 32)
    total = (c[:, -1] - c[:, 0]) % (1 << 32)
    med_total = float(np.median(total))
    stages = {s: {'median_cycles': float(np.median(d[:, i])), 'share': float(np.median(d[:, i])) / med_total} for i, s in enumerate(STAGES)}
    b.close()
    return {'metric': 'step-kernel stage cycles', 'lib': os.path.relpath(os.path.abspath(lib), REPO), 'envs': n, 'samples': int(c.shape[0]),
            'substep_median_cycles': med_total, 'stages': stages,
            'factor_plus_euler_solve_share': stages['factor_ld']['share'] + stages['euler_solve_m']['share'], 'device': smi}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--build', metavar='DIR')
    ap.add_argument('--lib')
    ap.add_argument('--ticks', type=int, default=20)
    ap.add_argument('--envs', type=int, default=4096)
    args = ap.parse_args()
    if args.build:
        print(build(args.build))
    if args.lib:
        print(json.dumps(run(args.lib, args.ticks, args.envs)), flush=True)


if __name__ == '__main__':
    main()
