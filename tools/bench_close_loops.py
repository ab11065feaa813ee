#!/usr/bin/env python3
"""bench_close_loops.py -- the cost of closing the legs' loops of a batch: cassie_batch_close_loops against the batch workaround it replaces.

  python tools/bench_close_loops.py [--reps R] [--passes P]

4096 fp32 environments of cassie.xml on torch's current stream, each started from the initial state with N(0, 0.05 rad) on every joint coordinate beyond
the pelvis and qvel ~ N(0, 0.5) (the start states of tests/test_close_loops.py).  Before every timed call the noisy state is copied back into the
batch's rows on the device; CUDA events bracket the timed work only.  Each figure is the median over P passes of the mean over R calls.

  close_loops_100% / _10%   one cassie_batch_close_loops launch with every / a tenth of the environments selected by a device mask (tol 1e-6 m)
  workaround_100%           as many rounds as the launch needed at most (its largest status iteration count) of: compute_dynamics (M and the connect
                            rows for every environment), a torch solve of the damped normal equations on the free columns, the step written into the
                            qvel rows and integrate_pos (which overwrites every environment's qpos); the velocity projection is not included

Prints one JSON line with the card's name and power limit, read in the same call."""
import argparse
import json
import os
import statistics
import subprocess
import sys

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [REPO, os.path.join(REPO, 'tests'), os.path.join(REPO, 'oracle')]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=50)
    ap.add_argument('--passes', type=int, default=3)
    args = ap.parse_args()
    import importlib
    import numpy as np
    import torch
    import loops_support as S
    P = importlib.import_module('cassie-mujoco-sim_b200')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    n = 4096
    torch.cuda.set_device(0)
    q, v, _ = S.start_states('cassie', 'noisy', n, 21, fp32=True)
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    b.set_qpos(q)
    b.set_qvel(v)
    qv, vv = b.torch_view('qpos'), b.torch_view('qvel')
    q0, v0 = qv.clone(), vv.clone()
    _, vfree = S.EmuLoops('cassie', True).free(q.shape[1], v.shape[1])
    free = torch.as_tensor(np.flatnonzero(vfree), device='cuda')
    gen = torch.Generator(device='cuda').manual_seed(3)
    masks = {100: torch.ones(n, dtype=torch.bool, device='cuda'), 10: torch.rand(n, device='cuda', generator=gen) < 0.1}

    def timed(work):
        total = 0.0
        for _ in range(args.reps):
            qv.copy_(q0)
            vv.copy_(v0)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            work()
            e1.record()
            e1.synchronize()
            total += e0.elapsed_time(e1)
        return total / args.reps

    out = dict(gpu=smi, n_env=n, precision='fp32', reps=args.reps, passes=args.passes, ms={})
    for pct, m in masks.items():
        def close(m=m):
            b.close_loops(m, max_iter=20, tol=1e-6)
        close()
        torch.cuda.synchronize()
        st = b.loop_status()
        if pct == 100:
            rounds = int(st['iterations'].max())
            out['iterations'] = dict(min=int(st['iterations'].min()), max=rounds, failed=int((st['iterations'] < 0).sum()))
        out['ms']['close_loops_%d%%' % pct] = round(statistics.median(timed(close) for _ in range(args.passes)), 4)

    b.compute_dynamics()
    dyn = b.torch_view('dyn')
    h = float(S.table('cassie')['timestep'][0])   # integrate_pos adds h qvel
    lam = torch.eye(12, device='cuda', dtype=dyn.dtype) * 1e-6

    def workaround():
        for _ in range(rounds):
            b.compute_dynamics()
            J = dyn[:, P.DYN['J_eq']].reshape(n, 12, P.DYN_COLS)[:, :, free]
            r = dyn[:, P.DYN['eq_err']]
            y = torch.linalg.solve(J @ J.transpose(1, 2) + lam, r.unsqueeze(2))
            step = -(J.transpose(1, 2) @ y).squeeze(2)
            vv.zero_()
            vv[:, free] = step / h
            b.integrate_pos()
    workaround()
    torch.cuda.synchronize()
    out['workaround_rounds'] = rounds
    out['ms']['workaround_100%'] = round(statistics.median(timed(workaround) for _ in range(args.passes)), 4)
    b.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
