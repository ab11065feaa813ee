"""Per-environment actuators on the fp64 oracle, for tests/test_env_actuators.py and tests/test_gpu_env_actuators.py.

The oracle gets ctrlrange and rpm through a temporary copy of its model table (MuJoCo's actuator_ctrlrange and actuator_user; nothing else in the table
changes).  It gets a torque delay d < 6 through its delay line, whose layout is the product's: before every call, slot 5 of each motor's line -- what
motor() applies -- is set to the torque of d ticks ago, which the line holds in slot d - 1 (the line then shifts as always, so its history is the
product's too).  For d = 0 it is set to this tick's torque, computed from the oracle's own closed blocks (o_pd_input_step, o_core_sim_step) and the
reference's motor() formula, and checked bit for bit against what motor() then shifts into slot 0.

The oracle's own source stays as it is (its delay length is the reference's compile-time constant); the delay is given to it from here instead.  The
d = 0 restatement calls the decoded closed blocks the oracle's default build runs, so ActOracle works on that build only, never on the archive-linked
one (oracle/_ref), whose closed blocks are the reference's objects."""
import ctypes as C
import math
import os
import tempfile

import numpy as np

from conftest import GOLDEN

NU, LINE = 10, 6


def table(model):
    """(gear [nu], ctrlrange [nu, 2], rpm [nu]) of the oracle's model table"""
    t = {ln.split()[0]: ln.split()[3:] for ln in open(os.path.join(GOLDEN, model + '.omodel')).read().split('\n') if ln.strip()}
    return (np.array([float(x) for x in t['actuator_gear']][:NU]), np.array([float(x) for x in t['actuator_ctrlrange']][:2 * NU]).reshape(NU, 2),
            np.array([float(x) for x in t['actuator_user']][:NU]))


class ActOracle:
    """one fp64 oracle environment with its own ctrlrange [nu, 2], rpm [nu] and delay [nu] (None: the model's; delay 6)"""

    def __init__(self, O, model, ctrlrange=None, rpm=None, delay=None):
        self.gear, cr0, rpm0 = table(model)
        self.cr = cr0 if ctrlrange is None else np.asarray(ctrlrange, float).reshape(NU, 2)
        self.rpm = rpm0 if rpm is None else np.asarray(rpm, float).reshape(NU)
        lines = open(os.path.join(GOLDEN, model + '.omodel')).read().split('\n')
        for i, ln in enumerate(lines):
            t = ln.split()
            if ln.startswith('actuator_ctrlrange '):
                lines[i] = ' '.join(t[:3] + [repr(float(x)) for x in self.cr.ravel()] + t[3 + 2 * NU:])
            elif ln.startswith('actuator_user '):
                lines[i] = ' '.join(t[:3] + [repr(float(x)) for x in self.rpm] + t[3 + NU:])
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, model + '.omodel')
            with open(p, 'w') as f:
                f.write('\n'.join(lines))
            self.o = O.OracleSim(p, ref=False)   # the decoded closed blocks, which tau_now restates
        self.O = O
        self.set_delay(np.full(NU, LINE) if delay is None else delay)
        self.line = np.ctypeslib.as_array(self.o.L.osim_torque_delay(self.o.h), shape=(NU, LINE))   # live view

    def set_delay(self, delay):
        self.delay = np.broadcast_to(np.asarray(delay, dtype=int), (NU,)).copy()
        assert np.all((self.delay >= 0) & (self.delay <= LINE))

    def tau_now(self, u):
        """the torque motor() will shift into slot 0 at the next call (the reference's :638-664 on the oracle's closed blocks)"""
        L, co = self.o.L, self.o.L.osim_cassie_out(self.o.h)
        tu, ti = (C.c_double * 10)(), (C.c_double * 10)()
        L.o_pd_input_step(C.byref(u), co, tu)
        L.o_core_sim_step(tu, co, ti)
        w = self.o.arr('actuator_velocity')
        out = np.zeros(NU)
        for i in range(NU):
            ratio, tmax, wmax = self.gear[i], self.cr[i][1], self.rpm[i] * 2 * math.pi / 60
            tlim = 2 * tmax * (1 - abs(w[i]) / wmax)
            tlim = max(min(tlim, tmax), 0.0)
            out[i] = math.copysign(min(abs(ti[i] / ratio), tlim), ti[i])
        return out

    def step_pd(self, u, y=None):
        now = self.tau_now(u) if np.any(self.delay == 0) else None
        for i in range(NU):
            d = self.delay[i]
            if d < LINE:
                self.line[i, 5] = now[i] if d == 0 else self.line[i, d - 1]
        self.o.step_pd(u, y)
        if now is not None:
            z = self.delay == 0
            assert np.array_equal(self.line[z, 0], now[z]), 'the restated motor() disagrees with the oracle'

    def drive_torque(self):
        """the drive torques of the last call's cassie_out: the applied ctrl times the gear, as motor() returns them"""
        return self.o.arr('ctrl')[:NU] * self.gear

    def close(self):
        self.o.close()


def saturating_pd(O, k, torque=None):
    """the motor-PD input of call k: targets swinging +-0.35 rad around the standing pose at 4 Hz with three times the standing gains, which drives
    the motors into their torque-speed limits; torque: an optional feed-forward [10]"""
    from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET
    s = 0.35 * math.sin(2 * math.pi * 4 * k * 5e-4)
    tgt = np.array(PD_TARGET) + s * np.array([0.3, 0.3, 1, -1, 0.5] * 2)
    return O.make_pd(torque=torque, pTarget=tgt, pGain=3 * np.array(PD_PGAIN, float), dGain=np.array(PD_DGAIN, float))


def pd_row(u):
    """the product's compact motor-PD row [50] (torque, pTarget, dTarget, pGain, dGain) of a pd_in_t's motorPd branch"""
    row = np.zeros(50)
    for j, name in enumerate(('torque', 'pTarget', 'dTarget', 'pGain', 'dGain')):
        for i in range(5):
            row[10 * j + i] = getattr(u.leftLeg.motorPd, name)[i]
            row[10 * j + 5 + i] = getattr(u.rightLeg.motorPd, name)[i]
    return row
