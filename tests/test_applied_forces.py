"""Per-environment applied forces (cassie_batch_set_applied_forces): the product's stepper source in the host emulation, with MuJoCo's xfrc_applied of
every body and qfrc_applied of every dof read from the environment's row (the F_XF instances), against the fp64 oracle given the same arrays.  The GPU
twins are in tests/test_gpu_applied_forces.py.

The emulation is tests/emu/emu_applied_forces.cpp, built into its own library here: the chain-twin source (extended, with model-valued contact,
mechanics, actuator and offset rows) and the plain-twin source (the plain kind, its scratch tail NaN-poisoned)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from mechanics_support import table

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
APPLIED_W, AP_XFRC, AP_QFRC, XFRC_W = 232, 0, 192, 8   # devmodel.h
CHAIN_PARENT, CHAIN, PLAIN, PLAIN_PARENT = 1, 2, 3, 4   # emu_xf_mode

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_applied_forces.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_applied_forces.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_xf_new.restype = vp
        L.emu_xf_new.argtypes = [C.c_char_p, ci]
        L.emu_xf_free.argtypes = [vp]
        L.emu_xf_mode.argtypes = [vp, ci]
        L.emu_xf_set_row.argtypes = [vp, dp]
        L.emu_xf_step.argtypes = [vp, dp, ci]
        L.emu_xf_bias.argtypes = [vp, dp]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


def to_row(xfrc, qfrc):
    """one environment's device row from xfrc_applied [nbody, 6] and qfrc_applied [nv] (dof columns: every shipped model has 32 main-tree dofs)"""
    row = np.zeros(APPLIED_W)
    row[AP_XFRC:AP_XFRC + xfrc.size] = np.ravel(xfrc)
    row[AP_QFRC:AP_QFRC + len(qfrc)] = qfrc
    return row


class XfSim:
    """one emulated environment running the source of `mode` (emu_xf_mode)"""

    def __init__(self, model, mode=CHAIN, fp32=False):
        self.L = lib()
        self.h = self.L.emu_xf_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h
        self.L.emu_xf_mode(self.h, mode)

    def close(self):
        if self.h:
            self.L.emu_xf_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def set_slot(self, wrench, body):
        row = np.zeros(XFRC_W)
        row[:6], row[6] = wrench, body
        assert self.L.emu_set(self.h, b'xfrc', _dp(row), XFRC_W) == XFRC_W

    def set_row(self, row):
        self.L.emu_xf_set_row(self.h, _dp(row))

    def step(self, nticks=1):
        self.L.emu_xf_step(self.h, _dp(PD_ROW), nticks)

    def bias(self, nv):
        out = np.zeros(64)
        assert self.L.emu_xf_bias(self.h, _dp(out)) == nv
        return out[:nv]


def pushed_bodies(model):
    """the bodies the schedule pushes: the pelvis, a foot, a tarsus, and the cup on the tray box (the extra free body)"""
    names = table(model)['names_body']
    return [names.index(b) for b in ('cassie-pelvis', 'left-foot', 'right-tarsus') + (('cup_box',) if model == 'cassie_tray_box' else ())]


def schedule(model, seed, nbody, nv):
    """wrenches redrawn every 100 ticks on every pushed body at once, random qfrc on every dof: a list of (xfrc [nbody, 6], qfrc [nv]) per 100 ticks"""
    rng = np.random.default_rng(seed)
    bodies = pushed_bodies(model)
    scale = {b: (f, t) for b, f, t in zip(bodies, (40.0, 8.0, 8.0, 0.6), (4.0, 0.8, 0.8, 0.02))}
    out = []
    for _ in range(5):
        x = np.zeros((nbody, 6))
        for b in bodies:
            x[b, :3] = rng.uniform(-1, 1, 3) * scale[b][0]
            x[b, 3:] = rng.uniform(-1, 1, 3) * scale[b][1]
        q = rng.uniform(-1, 1, nv) * 1.5
        if model == 'cassie_tray_box':
            q[32:35] *= 0.2   # the cup's translational dofs (a light body)
            q[35:38] *= 0.005
        out.append((x, q))
    return out


def oracle(oracle_mod, model):
    o = oracle_mod.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    o.set_caps()
    return o


# ------------------------------------------------------------------ 1. against the oracle: several bodies and every dof at once, with the slot
@pytest.mark.parametrize('mode', [CHAIN, PLAIN])
@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_hfield', 'cassie_tray_box'])
def test_applied_forces_follow_the_oracle(oracle_mod, model, mode):
    """fp64, 500 ticks: qpos within 1e-9 of the oracle with the same xfrc_applied / qfrc_applied, the same PGS iteration count every tick.  Bodies with
    a non-zero ipos are pushed, with torques, so a wrench applied at xpos, a torque taken in the body frame or a mishandled cup rotation shows"""
    o = oracle(oracle_mod, model)
    nb, nv = o.get_int('nbody'), o.nv
    e = XfSim(model, mode)
    ipos = table(model)['body_ipos'].reshape(-1, 3)
    assert all(np.linalg.norm(ipos[b]) > 1e-3 for b in pushed_bodies(model)[:3])
    slot = np.array([15.0, -10.0, 5.0, 1.0, -2.0, 0.5])
    pelvis = pushed_bodies(model)[0]
    e.set_slot(slot, pelvis)
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    worst, iters_equal = 0.0, True
    for k, (x, q) in enumerate(schedule(model, 11, nb, nv)):
        e.set_row(to_row(x, q))
        xo = x.copy()
        xo[pelvis] += slot   # the slot adds to its body's row entry
        o.arr('xfrc_applied')[:] = xo.ravel()
        o.arr('qfrc_applied')[:] = q
        for _ in range(100):
            o.step_pd(u)
            e.step()
            worst = max(worst, np.abs(e.get('qpos')[:o.nq] - o.arr('qpos')).max())
            iters_equal = iters_equal and int(e.get('counters')[3]) == o.get_int('solver_iter')
    print(model, mode, 'qpos %.2e' % worst)
    assert worst < 1e-9 and iters_equal, (model, mode, worst, iters_equal)
    # the forces change the motion
    o0 = oracle(oracle_mod, model)
    for _ in range(500):
        o0.step_pd(u)
    assert np.abs(o0.arr('qpos') - o.arr('qpos')).max() > 1e-3
    e.close()
    o.close()
    o0.close()


# ------------------------------------------------------------------ 2. zero rows are the parent instance
@pytest.mark.parametrize('pair', [(CHAIN_PARENT, CHAIN), (PLAIN_PARENT, PLAIN)])
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_zero_rows_reproduce_the_parent(model, pair):
    """f13c4 <-> f17c4 and f04 <-> f0404 sources: within 1e-12 in fp64 over 300 ticks, equal solver counters every tick"""
    a, b = XfSim(model, pair[0]), XfSim(model, pair[1])
    for k in range(300):
        a.step()
        b.step()
        assert np.abs(a.get('qpos') - b.get('qpos')).max() <= 1e-12, k
        assert np.array_equal(a.get('counters'), b.get('counters')), k
    a.close()
    b.close()


# ------------------------------------------------------------------ 3. one body's row is the slot
@pytest.mark.parametrize('body', ['cassie-pelvis', 'left-tarsus'])
def test_single_body_row_equals_the_slot(body):
    """the same wrench through the row of the chain twin and through the slot of its parent: within 1e-12 over 200 ticks"""
    model = 'cassie'
    b = table(model)['names_body'].index(body)
    w = np.array([30.0, -20.0, 10.0, 2.0, -1.0, 3.0]) * (1.0 if body == 'cassie-pelvis' else 0.2)
    nb = len(table(model)['names_body'])
    a, r = XfSim(model, CHAIN_PARENT), XfSim(model, CHAIN)
    a.set_slot(w, b)
    x = np.zeros((nb, 6))
    x[b] = w
    r.set_row(to_row(x, np.zeros(32)))
    worst = 0.0
    for k in range(200):
        a.step()
        r.step()
        worst = max(worst, np.abs(a.get('qpos') - r.get('qpos')).max())
        assert np.array_equal(a.get('counters'), r.get('counters')), k
    assert worst <= 1e-12, worst
    a.close()
    r.close()


def test_slot_reaches_the_extra_free_body(oracle_mod):
    """with rows, the slot pushes cassie_tray_box's cup, as MuJoCo's xfrc_applied does (its parent instance has no path to that body)"""
    model = 'cassie_tray_box'
    cup = table(model)['names_body'].index('cup_box')
    o = oracle(oracle_mod, model)
    e = XfSim(model, CHAIN)
    w = np.array([0.3, -0.2, 0.1, 0.004, -0.003, 0.002])
    e.set_slot(w, cup)
    o.arr('xfrc_applied')[6 * cup:6 * cup + 6] = w
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for _ in range(200):
        o.step_pd(u)
        e.step()
    assert np.abs(e.get('qpos')[:o.nq] - o.arr('qpos')).max() < 1e-9
    e.close()
    o.close()


# ------------------------------------------------------------------ 4. the dynamics launch keeps MuJoCo's qfrc_bias
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_dynamics_bias_excludes_applied_forces(oracle_mod, model):
    """mode 5 of the chain twin under pushes: its bias is the oracle's qfrc_bias at the same state (applied forces excluded), within 1e-9"""
    o = oracle(oracle_mod, model)
    nb, nv = o.get_int('nbody'), o.nv
    e = XfSim(model, CHAIN)
    x, q = schedule(model, 3, nb, nv)[0]
    e.set_row(to_row(x, q))
    o.arr('xfrc_applied')[:] = x.ravel()
    o.arr('qfrc_applied')[:] = q
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for _ in range(60):
        o.step_pd(u)
        e.step()
    nvm = 32
    bias = e.bias(nvm)
    o.forward()
    want = o.arr('qfrc_bias')[:nvm]
    assert np.abs(bias - want).max() < 1e-9 * max(1.0, np.abs(want).max()), np.abs(bias - want).max()
    e.close()
    o.close()
