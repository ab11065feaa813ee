"""Per-environment actuators (cassie_batch_set_env_actuators): the product's stepper source in the host emulation, with each motor's ctrlrange, no-load
speed and torque delay taken from the environment's row (the F_AC instances) instead of the model block.  The GPU twins are in
tests/test_gpu_env_actuators.py.

The emulation is tests/emu/emu_env_actuators.cpp, built into its own library here.  The fp64 oracle gets the same values through
tests/actuator_support.py: ctrlrange and rpm in a temporary copy of its model table, the delay through its delay line."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from actuator_support import LINE, NU, ActOracle, pd_row, saturating_pd, table
from conftest import PD_TARGET, REPO

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
OB_MTORQUE = 20   # devmodel.h: the observation's drive torques [10]
CS_DELAY = 84     # devmodel.h: the delay line [10][6] in the controller row

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_env_actuators.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_env_actuators.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_ac_new.restype = vp
        L.emu_ac_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_ac_free', 'emu_ac_forward'):
            getattr(L, n).argtypes = [vp]
        L.emu_ac_mode.argtypes = [vp, ci]
        L.emu_ac_set.argtypes = [vp, dp, dp, dp]
        L.emu_ac_row.argtypes = L.emu_ac_block.argtypes = [vp, dp]
        L.emu_ac_step.argtypes = [vp, dp, ci]
        L.emu_ac_delay_index.argtypes = [C.c_double, ci]
        L.emu_ac_check.argtypes = [ci, ci, vp, vp, vp, vp, C.c_char_p]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


class ActSim:
    """one emulated environment; mode 0 runs the extended F_ALL source, 1 the F_BP source with model-valued offset rows, 2 the F_BP | F_AC source"""

    def __init__(self, model, fp32=False, mode=2):
        self.L = lib()
        self.h = self.L.emu_ac_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h
        self.L.emu_ac_mode(self.h, mode)

    def close(self):
        if self.h:
            self.L.emu_ac_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def set_actuators(self, ctrlrange=None, rpm=None, delay=None):
        keep = [None if a is None else np.ascontiguousarray(a, dtype=np.float64).ravel() for a in (ctrlrange, rpm, delay)]
        self.L.emu_ac_set(self.h, *[_dp(a) for a in keep])

    def row(self):
        out = np.zeros(40)
        self.L.emu_ac_row(self.h, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def step(self, pd50, nticks=1):
        self.L.emu_ac_step(self.h, _dp(pd50), nticks)

    def forward(self):
        self.L.emu_ac_forward(self.h)

    def drive_torque(self):
        return self.get('obs')[OB_MTORQUE:OB_MTORQUE + NU]


def random_actuators(model, seed):
    """seeded per-motor values of the kinds users randomise: peak torque x [0.6, 1.2], no-load speed x [0.7, 1.3], delay uniform on 0..6"""
    _, cr, rpm = table(model)
    rng = np.random.default_rng(seed)
    return cr * rng.uniform(0.6, 1.2, (NU, 1)), rpm * rng.uniform(0.7, 1.3, NU), rng.integers(0, LINE + 1, NU)


# ------------------------------------------------------------------ 1. rows at the model's values are the F_BP source, bitwise
@pytest.mark.parametrize('fp32', [False, True])
def test_model_rows_are_bitwise_the_body_pos_source(oracle_mod, fp32):
    a, b = ActSim('cassie', fp32, mode=1), ActSim('cassie', fp32, mode=2)
    _, cr, rpm = table('cassie')
    b.set_actuators(cr, rpm, np.full(NU, LINE))   # what the setter stores for the model's values
    blk = np.zeros(30)
    b.L.emu_ac_block(b.h, blk.ctypes.data_as(C.POINTER(C.c_double)))
    assert np.array_equal(b.row()[:30], blk)      # lo, hi and wmax are the block's act_ctrl_lo / act_ctrl_hi / act_wmax bit for bit
    for k in range(400):
        u = pd_row(saturating_pd(oracle_mod, k))
        a.step(u)
        b.step(u)
        for f in ('qpos', 'qvel', 'obs', 'aux', 'cst', 'counters'):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    a.close()
    b.close()


# ------------------------------------------------------------------ 2. against the oracle
@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box'])
def test_env_actuators_follow_the_oracle(oracle_mod, model):
    """fp64: per-motor ctrlrange / rpm / delay; qpos and the observation's drive torques within 1e-9 of the oracle given the same values over 500
    saturating ticks, the same PGS iteration count every tick"""
    cr, rpm, dl = random_actuators(model, 11)
    dl[:3] = [0, 3, 6]   # every kind of delay in every run
    cr[::2, 0] = -0.3 * cr[::2, 1]   # asymmetric ranges on half the motors: the actuation's lower clamp acts
    o = ActOracle(oracle_mod, model, cr, rpm, dl)
    e = ActSim(model)
    e.set_actuators(cr, rpm, dl)
    worst_q, worst_t, iters_equal, saturated, below = 0.0, 0.0, True, 0, 0
    for k in range(500):
        u = saturating_pd(oracle_mod, k)
        o.step_pd(u)
        e.step(pd_row(u))
        worst_q = max(worst_q, np.abs(e.get('qpos')[:o.o.nq] - o.o.arr('qpos')).max())
        worst_t = max(worst_t, np.abs(e.drive_torque() - o.drive_torque()).max())
        iters_equal = iters_equal and int(e.get('counters')[3]) == o.o.get_int('solver_iter')
        saturated += int(np.sum(np.isclose(np.abs(o.drive_torque()), o.cr[:, 1] * o.gear, rtol=0, atol=1e-12)))
        below += int(np.sum(o.o.arr('ctrl')[:NU] < cr[:, 0]))
    print(model, 'qpos %.2e, drive torque %.2e, %d saturated motor-ticks, %d clamped at lo' % (worst_q, worst_t, saturated, below))
    assert worst_q < 1e-9 and worst_t < 1e-9 and iters_equal, (model, worst_q, worst_t, iters_equal)
    assert saturated > 0 and below > 0   # the inputs reached the rows' peak torques, and the lower clamps acted
    # the values change the motion: the model's actuators give another trajectory
    o0 = ActOracle(oracle_mod, model)
    for k in range(500):
        o0.step_pd(saturating_pd(oracle_mod, k))
    assert np.abs(o0.o.arr('qpos') - o.o.arr('qpos')).max() > 1e-5
    e.close()
    o.close()
    o0.close()


# ------------------------------------------------------------------ 3. the delay
def _impulse_run(oracle_mod, make, d, k0, on):
    """the drive torques of motor 3 over 20 calls with zero PD gains and a 20 Nm feed-forward on it from call k0 (on) or never"""
    s = make(d)
    out = []
    for k in range(20):
        tq = np.zeros(NU)
        if on and k >= k0:
            tq[3] = 20.0
        u = oracle_mod.make_pd(torque=tq, pTarget=PD_TARGET)
        if isinstance(s, ActOracle):
            s.step_pd(u)
            out.append(s.drive_torque()[3])
        else:
            s.step(pd_row(u))
            out.append(s.drive_torque()[3])
    s.close()
    return np.array(out)


@pytest.mark.parametrize('d', range(LINE + 1))
def test_delay_impulse(oracle_mod, d):
    """a step of feed-forward torque at call k shows in the drive torque first at call k + d -- against the same run without the step (the safety
    layer's limit springs can make the torque non-zero before k); the delayed oracle shows it at the same call, with the same values"""
    k0 = 5
    _, cr, rpm = table('cassie')

    def emu(dd):
        s = ActSim('cassie')
        s.set_actuators(cr, rpm, np.full(NU, dd))
        return s

    def orc(dd):
        return ActOracle(oracle_mod, 'cassie', delay=np.full(NU, dd))

    for make in (emu, orc):
        a, b = _impulse_run(oracle_mod, make, d, k0, True), _impulse_run(oracle_mod, make, d, k0, False)
        first = int(np.flatnonzero(a != b)[0])
        assert first == k0 + d, (make.__name__, d, first)
    assert np.abs(_impulse_run(oracle_mod, emu, d, k0, True) - _impulse_run(oracle_mod, orc, d, k0, True)).max() < 1e-9


def test_delay_switch(oracle_mod):
    """from 6 to 2 mid-run: the next call applies the torque of two calls earlier at once (slot 1 of the line before the call), and the run follows
    the oracle with the same switch"""
    e, o = ActSim('cassie'), ActOracle(oracle_mod, 'cassie')
    _, cr, rpm = table('cassie')
    e.set_actuators(cr, rpm, np.full(NU, LINE))
    gear = o.gear
    worst = 0.0
    for k in range(300):
        if k == 150:
            e.set_actuators(delay=np.full(NU, 2))
            o.set_delay(2)
            line = e.get('cst')[CS_DELAY:CS_DELAY + 60].reshape(NU, LINE).copy()
        u = saturating_pd(oracle_mod, k)
        o.step_pd(u)
        e.step(pd_row(u))
        if k == 150:
            assert np.array_equal(e.drive_torque(), line[:, 1] * gear)
            assert not np.array_equal(line[:, 1], line[:, 5])
        worst = max(worst, np.abs(e.get('qpos')[:o.o.nq] - o.o.arr('qpos')).max(), np.abs(e.drive_torque() - o.drive_torque()).max())
    assert worst < 1e-9, worst
    e.close()
    o.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_stored_delays_outside_the_line(oracle_mod, fp32):
    """a row written through the device pointer can hold anything: -3, 9 and NaN act as 0, 6 and 0 (clamped before the conversion), bit for bit"""
    L = lib()
    assert [L.emu_ac_delay_index(v, int(fp32)) for v in (-3.0, 9.0, float('nan'), 0.0, 2.7, 6.0, -0.5, 1e30)] == [0, 6, 0, 0, 2, 6, 0, 6]
    _, cr, rpm = table('cassie')
    odd, even = np.array([-3, 9, np.nan] * 3 + [9.0]), np.array([0, 6, 0] * 3 + [6.0])
    a, b = ActSim('cassie', fp32), ActSim('cassie', fp32)
    a.set_actuators(cr, rpm, odd)
    b.set_actuators(cr, rpm, even)
    for k in range(200):
        u = pd_row(saturating_pd(oracle_mod, k))
        a.step(u)
        b.step(u)
    for f in ('qpos', 'qvel', 'obs', 'cst'):
        assert np.array_equal(a.get(f), b.get(f)), f
    a.close()
    b.close()


# ------------------------------------------------------------------ 4. the setter's check
def test_setter_refusals():
    """the batch setter's check: every masked value before anything changes; unmasked environments are not checked"""
    L = lib()
    n = 3
    _, cr0, rpm0 = table('cassie')
    cr, rpm, dl = np.tile(cr0, (n, 1, 1)), np.tile(rpm0, (n, 1)), np.full((n, NU), 6, dtype=np.int32)

    def check(cr_, rpm_, dl_, mask=None):
        why = C.create_string_buffer(256)
        arr = [None if a is None else np.ascontiguousarray(a) for a in (cr_, rpm_, dl_)]
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        r = L.emu_ac_check(n, NU, *[None if a is None else a.ctypes.data_as(C.c_void_p) for a in arr], None if m is None else m.ctypes.data_as(C.c_void_p), why)
        return r, why.value.decode()

    assert check(cr, rpm, dl)[0] == 0
    assert check(None, None, None)[0] == 0
    bad = []
    c = cr.copy(); c[1, 4, 0] = np.nan; bad.append((c, rpm, dl, 'not finite'))
    c = cr.copy(); c[2, 0] = [1.0, 1.0]; bad.append((c, rpm, dl, 'lo < hi'))
    c = cr.copy(); c[0, 3] = [2.0, -2.0]; bad.append((c, rpm, dl, 'lo < hi'))
    r_ = rpm.copy(); r_[1, 2] = 0.0; bad.append((cr, r_, dl, 'rpm'))
    r_ = rpm.copy(); r_[1, 2] = np.inf; bad.append((cr, r_, dl, 'rpm'))
    d_ = dl.copy(); d_[2, 9] = 7; bad.append((cr, rpm, d_, 'delay'))
    d_ = dl.copy(); d_[0, 0] = -1; bad.append((cr, rpm, d_, 'delay'))
    for c, r_, d_, word in bad:
        r, why = check(c, r_, d_)
        assert r == 1 and word in why and 'environment' in why, (word, why)
    # a refused value in an unselected environment is not looked at
    c = cr.copy(); c[1, 4, 0] = np.nan
    assert check(c, rpm, dl, mask=[1, 0, 1])[0] == 0
    assert check(c, rpm, dl, mask=[0, 1, 0])[0] == 1
