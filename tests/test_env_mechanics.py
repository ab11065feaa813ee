"""Per-environment mechanics (cassie_batch_set_env_mechanics): the product's stepper source in the host emulation, with each body's principal inertia,
each dof's armature and each hinge's spring taken from the environment's row (the F_MC instances) instead of the model block.  The GPU twins are in
tests/test_gpu_env_mechanics.py.

The emulation is tests/emu/emu_env_mechanics.cpp, built into its own library here.  The fp64 oracle gets the same values through a temporary copy of its
model table (tests/mechanics_support.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from mechanics_support import HINGE, changeable_bodies, model_values, oracle_with, random_mechanics, table

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
CE_BINVW, CE_DINVW, CE_PGS = 192, 224, 258   # devmodel.h CE_*
MC_INERTIA, MC_ARMATURE, MC_STIFF, MC_SPRING, MECH_W = 0, 96, 128, 160, 192   # devmodel.h MC_*

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_env_mechanics.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_env_mechanics.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_mc_new.restype = vp
        L.emu_mc_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_mc_free', 'emu_mc_forward', 'emu_mc_set_const'):
            getattr(L, n).argtypes = [vp]
        L.emu_mc_mode.argtypes = [vp, ci]
        L.emu_mc_set.argtypes = [vp, dp, dp, dp, dp]
        L.emu_mc_poke.argtypes = [vp, ci, C.c_double]
        L.emu_mc_row.argtypes = [vp, dp]
        L.emu_mc_model.argtypes = [vp, dp, dp, dp, dp]
        L.emu_mc_step.argtypes = [vp, dp, ci]
        L.emu_mc_check.argtypes = [vp, ci, vp, vp, vp, vp, vp, C.c_char_p]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


class MechSim:
    """one emulated environment; mode 0 runs the extended F_ALL source, 1 the F_AC source with model-valued rows, 2 the F_AC | F_MC source"""

    def __init__(self, model, fp32=False, mode=2):
        self.L = lib()
        self.h = self.L.emu_mc_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h
        self.L.emu_mc_mode(self.h, mode)
        self.name = model

    def close(self):
        if self.h:
            self.L.emu_mc_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def set_mechanics(self, inertia=None, armature=None, stiffness=None, springref=None):
        self._keep = [None if a is None else np.ascontiguousarray(a, dtype=np.float64).ravel() for a in (inertia, armature, stiffness, springref)]
        self.L.emu_mc_set(self.h, *[_dp(a) for a in self._keep])

    def model(self):
        """(inertia [nbody, 3], armature [nv], stiffness [njnt], springref [njnt]) of the product's compiled model, what the batch's get reports without
        rows (the oracle's table may differ in the last digits)"""
        nb, nv, nj = (len(table(self.name)[k]) for k in ('body_weldid', 'dof_armature', 'jnt_type'))
        out = [np.zeros((nb, 3)), np.zeros(nv), np.zeros(nj), np.zeros(nj)]
        self.L.emu_mc_model(self.h, *[_dp(v) for v in out])
        return out

    def row(self):
        out = np.zeros(MECH_W)
        self.L.emu_mc_row(self.h, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def step(self, pd50, nticks=1):
        self.L.emu_mc_step(self.h, _dp(pd50), nticks)

    def forward(self):
        self.L.emu_mc_forward(self.h)

    def set_const(self):
        self.L.emu_mc_set_const(self.h)


# ------------------------------------------------------------------ 1. rows at the model's values are the F_AC source, bitwise
@pytest.mark.parametrize('fp32', [False, True])
def test_model_rows_are_bitwise_the_actuator_source(fp32):
    a, b = MechSim('cassie', fp32, mode=1), MechSim('cassie', fp32, mode=2)
    b.set_mechanics(*b.model())   # what the setter stores for the model's values
    for k in range(400):
        a.step(PD_ROW)
        b.step(PD_ROW)
        for f in ('qpos', 'qvel', 'obs', 'aux', 'cst', 'counters'):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    a.close()
    b.close()


# ------------------------------------------------------------------ 2. against the oracle
@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box'])
def test_env_mechanics_follow_the_oracle(oracle_mod, model):
    """fp64: qpos within 1e-9 of the oracle with the same body_inertia, dof_armature, jnt_stiffness and qpos_spring over 500 ticks, the same PGS iteration
    count every tick"""
    I, arm, k, q = random_mechanics(model, 21)
    o = oracle_with(oracle_mod, model, I, arm, k, q)
    e = MechSim(model)
    e.set_mechanics(I, arm, k, q)
    e.forward()
    o.forward()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    worst, iters_equal = 0.0, True
    for _ in range(500):
        o.step_pd(u)
        e.step(PD_ROW)
        worst = max(worst, np.abs(e.get('qpos')[:o.nq] - o.arr('qpos')).max())
        iters_equal = iters_equal and int(e.get('counters')[3]) == o.get_int('solver_iter')
    print(model, 'qpos %.2e' % worst)
    assert worst < 1e-9 and iters_equal, (model, worst, iters_equal)
    # the values change the motion: the model's own trajectory is elsewhere
    o0 = oracle_with(oracle_mod, model)
    for _ in range(500):
        o0.step_pd(u)
    assert np.abs(o0.arr('qpos') - o.arr('qpos')).max() > 1e-5
    e.close()
    o.close()
    o0.close()


@pytest.mark.parametrize('part', ['inertia', 'armature', 'springs'])
def test_each_part_follows_the_oracle(oracle_mod, part):
    """each part alone (the others the model's) moves the trajectory, and the oracle given that part alone follows it"""
    I0, a0, k0, q0 = model_values('cassie')   # the oracle's table: the emulation gets the same values
    I, arm, k, q = random_mechanics('cassie', 33)
    vals = dict(inertia=(I, a0, k0, q0), armature=(I0, arm, k0, q0), springs=(I0, a0, k, q))[part]
    o, o0 = oracle_with(oracle_mod, 'cassie', *vals), oracle_with(oracle_mod, 'cassie')
    e = MechSim('cassie')
    e.set_mechanics(*vals)
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    worst = 0.0
    for _ in range(300):
        o.step_pd(u)
        o0.step_pd(u)
        e.step(PD_ROW)
        worst = max(worst, np.abs(e.get('qpos')[:o.nq] - o.arr('qpos')).max())
    assert worst < 1e-9, (part, worst)
    assert np.abs(o0.arr('qpos') - o.arr('qpos')).max() > 1e-7, part
    for s in (e, o, o0):
        s.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box'])
def test_set_const_rows_follow_the_oracle(oracle_mod, model):
    """mode 3 at qpos0 with the environment's inertia and armature: the invweights and the PGS scale match the oracle's mj_setConst with the same table"""
    I, arm, k, q = random_mechanics(model, 9)
    o = oracle_with(oracle_mod, model, I, arm, k, q)
    e = MechSim(model)
    e.set_mechanics(I, arm, k, q)
    e.set_const()
    o.just_set_const()
    nb, nv = o.get_int('nbody'), o.get_int('nv')
    xb = nb - 1 if model == 'cassie_tray_box' else -1
    c = e.get('cenv')
    bi = [b for b in range(nb) if b != xb]
    assert np.abs(c[CE_BINVW:CE_BINVW + nb][bi] - o.model_arr('body_invweight0')[0::2][bi]).max() < 1e-12
    assert np.abs(c[CE_DINVW:CE_DINVW + 32] / o.model_arr('dof_invweight0')[:32] - 1).max() < 1e-12
    assert abs(c[CE_PGS] * o.model_arr('meaninertia')[0] * nv - 1) < 1e-12
    # and they differ from the model's constants
    ref = oracle_with(oracle_mod, model)
    ref.just_set_const()
    assert np.abs(ref.model_arr('dof_invweight0') - o.model_arr('dof_invweight0')).max() > 1e-9
    assert abs(ref.model_arr('meaninertia')[0] - o.model_arr('meaninertia')[0]) > 1e-9
    e.close()
    o.close()
    ref.close()


# ------------------------------------------------------------------ 3. the row's layout and the hold
def test_row_layout():
    t = table('cassie')
    I, arm, k, q = random_mechanics('cassie', 4)
    e = MechSim('cassie')
    e.set_mechanics(I, arm, k, q)
    r = e.row()
    nb = len(t['body_weldid'])
    assert np.array_equal(r[MC_INERTIA:MC_INERTIA + 3 * nb], I.ravel()) and not r[MC_INERTIA + 3 * nb:MC_ARMATURE].any()
    assert np.array_equal(r[MC_ARMATURE:MC_ARMATURE + 32], arm[:32])
    for j, d in enumerate(t['jnt_dofadr']):
        if t['jnt_type'][j] == HINGE:
            assert r[MC_STIFF + d] == k[j] and r[MC_SPRING + d] == q[j], j
    e.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_slide_slots_are_not_read(fp32):
    """a stiffness and rest position written into a slide dof's slots (the pelvis slides, where cassie_sim_hold puts its spring) change nothing, bit for
    bit; the same values in a hinge's slots do"""
    t = table('cassie')
    a, b, c = (MechSim('cassie', fp32) for _ in range(3))
    for s in (a, b, c):
        s.set_mechanics(*s.model())
    for d in range(3):   # the pelvis slides' dofs
        assert t['jnt_type'][t['dof_jntid'][d]] == 2
        b.L.emu_mc_poke(b.h, MC_STIFF + d, 1e5)
        b.L.emu_mc_poke(b.h, MC_SPRING + d, 0.3)
    shin = t['jnt_dofadr'][list(t['jnt_stiffness']).index(1500.0)]
    c.L.emu_mc_poke(c.h, MC_STIFF + shin, 1e5)
    for _ in range(100):
        for s in (a, b, c):
            s.step(PD_ROW)
    for f in ('qpos', 'qvel', 'obs', 'counters'):
        assert np.array_equal(a.get(f), b.get(f)), f
    assert not np.array_equal(a.get('qpos'), c.get('qpos'))
    for s in (a, b, c):
        s.close()


# ------------------------------------------------------------------ 4. the setter's check
def _check(s, n, parts, mask=None):
    why = C.create_string_buffer(512)
    arr = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in parts]
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    r = s.L.emu_mc_check(s.h, n, *[None if a is None else a.ctypes.data_as(C.c_void_p) for a in arr], None if m is None else m.ctypes.data_as(C.c_void_p), why)
    return r, why.value.decode()


@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_setter_refusals(model):
    """the batch setter's check: every masked value before anything changes, with the environment, the body / dof / joint and the field named; unmasked
    environments are not checked"""
    n = 3
    t = table(model)
    s = MechSim(model)
    base = [np.tile(v, (n,) + (1,) * v.ndim) for v in s.model()]
    assert _check(s, n, base)[0] == 0
    assert _check(s, n, [None] * 4)[0] == 0
    # accepted: changeable bodies, main-tree armature, hinge springs (within the rules)
    ok = [v.copy() for v in base]
    b = changeable_bodies(model)[0]
    ok[0][1, b] *= 1.3
    ok[1][2, 7] = 0.0
    ok[2][0, :] = np.where(t['jnt_type'] == HINGE, 0.0, ok[2][0])
    assert _check(s, n, ok)[0] == 0, _check(s, n, ok)[1]

    def bad(part, env, idx, value, words):
        p = [v.copy() for v in base]
        p[part][(env,) + idx] = value
        r, why = _check(s, n, p)
        assert r == 1 and all(w in why for w in words) and 'environment %d' % env in why, (part, idx, value, why)
        m = [1] * n
        m[env] = 0
        assert _check(s, n, p, mask=m)[0] == 0   # a refused value in an unselected environment is not looked at

    names = t['names_body']
    bad(0, 1, (b, 0), np.nan, ['body_inertia', 'not finite', names[b]])
    bad(0, 2, (b, 1), -1e-3, ['body_inertia', '>= 0'])
    I = base[0][0, b]
    bad(0, 0, (b,), [I.max() * 3, I.max(), I.max()], ['A + B >= C'])
    bad(0, 1, (0,), [1.0, 1.0, 1.0], ['world body'])
    welded = [x for x in range(1, len(t['body_weldid'])) if t['body_weldid'][x] == 0]
    for w in welded:
        bad(0, 1, (w,), base[0][0, w] * 1.1 + 1e-3, ['welded to the world'])
    bad(1, 1, (7,), np.inf, ['dof_armature', 'not finite', 'dof 7'])
    bad(1, 2, (6,), -0.01, ['dof_armature', '>= 0'])
    hinge = [j for j in range(len(t['jnt_type'])) if t['jnt_type'][j] == HINGE]
    slide = [j for j in range(len(t['jnt_type'])) if t['jnt_type'][j] == 2]
    ball = [j for j in range(len(t['jnt_type'])) if t['jnt_type'][j] == 1]
    bad(2, 0, (hinge[3],), np.nan, ['jnt_stiffness', 'not finite'])
    bad(2, 0, (hinge[3],), -5.0, ['jnt_stiffness', '>= 0'])
    bad(3, 1, (hinge[3],), np.inf, ['qpos_spring', 'not finite'])
    for j in slide + ball:
        bad(2, 2, (j,), 100.0, ['jnt_stiffness', 'slide, ball or free'])
        bad(3, 2, (j,), 0.5, ['qpos_spring', 'slide, ball or free'])
    if model == 'cassie_tray_box':
        xb = len(t['body_weldid']) - 1
        bad(0, 1, (xb,), base[0][0, xb] * 1.1, ['extra free body'])
        bad(1, 1, (33,), 0.1, ['extra free body'])
        free = [j for j in range(len(t['jnt_type'])) if t['jnt_type'][j] == 0]
        bad(2, 0, (free[0],), 10.0, ['slide, ball or free'])
    s.close()
