#!/usr/bin/env python3
"""bench_ik.py -- the cost of posing a batch's feet: cassie_batch_solve_ik against the host loop it replaces.

  python tools/bench_ik.py [--reps R] [--passes P]

4096 fp32 environments of cassie.xml on torch's current stream, each started from a settled standing pose, with two foot targets (the left-foot-pt and
right-foot-pt sites in the pelvis frame: position plus the foot's pitch and yaw) taken from reachable poses -- the standing motors plus U(-0.3, 0.3) rad,
clipped to their ranges, closed by close_loops' source in fp64 (tests/ik_support.py).  Before every timed call the standing state is copied back into
the batch's rows on the device; CUDA events bracket the timed work only.  Each figure is the median over P passes of the mean over R calls.

  solve_ik_100% / _10%   one cassie_batch_solve_ik launch with every / a tenth of the environments selected by a device mask
  host_loop_100%         as many rounds as the launch needed at most of: frame_jacobian for each target (a launch and a synchronous copy each),
                         compute_dynamics (the connect rows), forward (the frame poses), a torch damped least-squares solve of the position rows
                         stacked with the connect rows on the free columns, the step clamped to the motor ranges, written into the qvel rows and
                         applied by integrate_pos, then close_loops; the orientation rows and the velocity stage are not included

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
    ap.add_argument('--reps', type=int, default=20)
    ap.add_argument('--passes', type=int, default=3)
    args = ap.parse_args()
    import importlib
    import numpy as np
    import torch
    import ik_support as S
    P = importlib.import_module('cassie-mujoco-sim_b200')
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    n, model = 4096, 'cassie'
    torch.cuda.set_device(0)
    spec = S.feet(model)
    start, posed = S.reachable(model, 256, 41, fp32=True)
    tg = S.target_rows(model, spec, posed)
    rep = np.arange(n) % 256
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    b.set_qpos(start[rep])
    b.set_qvel(np.zeros((n, b.nv)))
    b.set_ik([s['name'] for s in spec], [s['kind'] for s in spec], [s['frame'] for s in spec], [s['w'] for s in spec])
    b.set_frames([s['name'] for s in spec], [s['kind'] for s in spec])
    b.torch_view('ik_targets').copy_(torch.as_tensor(tg[rep], device='cuda'))
    qv, vv = b.torch_view('qpos'), b.torch_view('qvel')
    q0, v0 = qv.clone(), vv.clone()
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

    out = dict(gpu=smi, n_env=n, precision='fp32', targets=2, reps=args.reps, passes=args.passes, ms={})
    for pct, m in masks.items():
        def solve(m=m):
            b.solve_ik(m)
        solve()
        torch.cuda.synchronize()
        st = b.ik_status()
        if pct == 100:
            rounds = int(st['iterations'].max())
            out['iterations'] = dict(min=int(st['iterations'].min()), max=rounds, reached=int((st['outcome'] == 1).sum()), best_effort=int((st['outcome'] == 2).sum()),
                                     kept=int((st['outcome'] == -1).sum()), pos_residual_max=float(st['pos_residual'].max()), ori_residual_max=float(st['ori_residual'].max()))
        out['ms']['solve_ik_%d%%' % pct] = round(statistics.median(timed(solve) for _ in range(args.passes)), 4)

    dof, lim, lo, hi = S.EmuIk(model, True).columns()
    free = torch.as_tensor(dof.astype(np.int64), device='cuda')
    lo_t, hi_t = torch.as_tensor(np.where(lim, lo, -np.inf), device='cuda', dtype=torch.float32), torch.as_tensor(np.where(lim, hi, np.inf), device='cuda', dtype=torch.float32)
    t = S.LS.table(model)
    jq = torch.as_tensor(np.array([int(t['jnt_qposadr'][int(t['dof_jntid'][d])]) for d in dof]), device='cuda')
    hinge = torch.as_tensor(np.array([int(t['jnt_type'][int(t['dof_jntid'][d])]) != 1 for d in dof]), device='cuda')
    h = float(t['timestep'][0])
    tgw = S.target_rows(model, S.feet(model, frame=S.WORLD), posed)   # the pelvis is held: the same targets in world axes
    tgt = torch.as_tensor(tgw[rep][:, :2, :3], device='cuda', dtype=torch.float32)
    lam = 1e-4
    b.compute_dynamics()
    dyn = b.torch_view('dyn')

    def host_loop():
        for _ in range(rounds):
            J = [torch.as_tensor(b.frame_jacobian(k)[0], device='cuda', dtype=torch.float32) for k in range(2)]   # world jacp [n, 3, nv]
            b.compute_dynamics()
            b.forward()
            fr = b.torch_view('frames').view(n, 2, P.FRAME_WIDTH)
            err = torch.cat([fr[:, k, :3] - tgt[:, k] for k in range(2)], 1)
            Jt = torch.cat([j[:, :, free] for j in J], 1)
            Jc = dyn[:, P.DYN['J_eq']].reshape(n, 12, P.DYN_COLS)[:, :, free]
            A = torch.cat([Jt, Jc], 1)
            r = torch.cat([err, dyn[:, P.DYN['eq_err']]], 1)
            dq = -(A.transpose(1, 2) @ torch.linalg.solve(A @ A.transpose(1, 2) + lam * torch.eye(A.shape[1], device='cuda'), r.unsqueeze(2))).squeeze(2)
            cur = qv[:, jq]
            dq = torch.where(hinge, torch.clamp(cur + dq, lo_t, hi_t) - cur, dq)
            vv.zero_()
            vv[:, free] = dq / h
            b.integrate_pos()
            b.close_loops(None)
    host_loop()
    torch.cuda.synchronize()
    out['host_loop_rounds'] = rounds
    out['ms']['host_loop_100%'] = round(statistics.median(timed(host_loop) for _ in range(args.passes)), 4)
    b.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
