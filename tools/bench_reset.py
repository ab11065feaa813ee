#!/usr/bin/env python3
"""bench_reset.py -- the cost of resetting environments of a batch: the host verbs against the device-masked restore (cassie_batch_reset_where).

  python tools/bench_reset.py [--reps R] [--ticks T] [--passes P] [--package DIR]

4096 fp32 environments of cassie.xml with configuration 2's controller (the standing motor-PD rows), on torch's current stream, settled 300 ticks; the
reset bank holds 64 environments of that settled state.  Each figure is the median of P passes.

Per call, with 1 % and 10 % of the environments selected by a mask that lives on the device (R calls, host clock around work ending in a device
synchronise):
  host_reset         the mask copied to the host (a synchronising copy), then cassie_batch_reset(mask)
  host_set_state     cassie_batch_set_state(snapshot, mask) with a host mask
  reset_where        cassie_batch_reset_where(mask, entries)
  reset_forward      cassie_batch_reset_where, then cassie_batch_forward_where(mask)
RL loop: T ticks of step(1), each environment done when its own 300-tick time limit runs out (the limits staggered over the batch: about 14 resets per
tick), then either the host path (mask to the host, cassie_batch_reset(mask)) or reset_where with entries from torch.randint; env-steps per second.

--package DIR imports the package from DIR instead of this repository (e.g. an older build): the arms its library lacks are skipped.
Prints one JSON line with the card's name and power limit."""
import argparse
import importlib.util
import json
import os
import statistics
import subprocess
import sys
import time

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(REPO, 'tests'))


def load_package(path):
    spec = importlib.util.spec_from_file_location('cassie_b200_bench', os.path.join(path, '__init__.py'), submodule_search_locations=[path])
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--reps', type=int, default=200)
    ap.add_argument('--ticks', type=int, default=1000)
    ap.add_argument('--passes', type=int, default=3)
    ap.add_argument('--package', default=os.path.join(REPO, 'cassie-mujoco-sim_b200'))
    args = ap.parse_args()
    import numpy as np
    import torch
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    P = load_package(os.path.abspath(args.package))
    smi = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], capture_output=True, text=True).stdout.strip()
    n, K, limit = 4096, 64, 300
    torch.cuda.set_device(0)
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    b.set_stream(torch.cuda.current_stream().cuda_stream)   # torch's mask and entry writes are ordered before the batch's launches
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.reset()
    b.step(limit)
    snap = b.get_state()
    device_verbs = hasattr(P.CassieBatch, 'reset_where') and hasattr(b.L, 'cassie_batch_reset_where')
    if device_verbs:
        b.set_reset_bank(snap, np.random.default_rng(1).choice(n, K, replace=False))
    gen = torch.Generator(device='cuda').manual_seed(2)

    def timed(fn, reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for _ in range(reps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) / reps * 1e3

    out = dict(gpu=smi, n_env=n, bank=K, reps=args.reps, passes=args.passes, per_call_ms={}, rl_loop={})
    for frac in (0.01, 0.10):
        mask = torch.rand(n, device='cuda', generator=gen) < frac
        entry = torch.randint(0, K, (n,), device='cuda', dtype=torch.int32, generator=gen)
        m_host = mask.cpu().numpy().astype(np.uint8)
        arms = dict(host_reset=lambda: b.reset(mask.cpu().numpy().astype(np.uint8)), host_set_state=lambda: b.set_state(snap, m_host))
        if device_verbs:
            arms['reset_where'] = lambda: b.reset_where(mask, entry)
            arms['reset_forward'] = lambda: (b.reset_where(mask, entry), b.forward_where(mask))
        for name, fn in arms.items():
            fn()
            out['per_call_ms']['%s_%d%%' % (name, round(frac * 100))] = round(statistics.median(timed(fn, args.reps) for _ in range(args.passes)), 4)

    def loop(path):
        b.set_state(snap)
        ticks = (torch.arange(n, device='cuda', dtype=torch.int32) * limit) // n   # staggered time limits
        resets = 0

        def tick():
            nonlocal resets, ticks
            b.step(1)
            ticks = ticks + 1
            done = ticks >= limit
            ticks = torch.where(done, torch.zeros_like(ticks), ticks)
            if path == 'host':
                m = done.cpu().numpy()
                resets += int(m.sum())
                b.reset(m.astype(np.uint8))
            else:
                b.reset_where(done, torch.randint(0, K, (n,), device='cuda', dtype=torch.int32, generator=gen))
        for _ in range(20):
            tick()
        resets = 0
        ms = timed(tick, args.ticks)
        return n / (ms * 1e-3), resets / args.ticks

    for path in (('host', 'device') if device_verbs else ('host',)):
        runs = [loop(path) for _ in range(args.passes)]
        rate = statistics.median(r[0] for r in runs)
        out['rl_loop'][path] = dict(env_steps_per_s=round(rate), ms_per_tick=round(n / rate * 1e3, 4))
        if path == 'host':
            out['rl_loop'][path]['resets_per_tick'] = round(runs[0][1], 2)
    b.free_state(snap)
    b.close()
    print(json.dumps(out))


if __name__ == '__main__':
    main()
