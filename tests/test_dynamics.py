"""Dynamics rows (cassie_batch_dynamics, launch mode 5): the product's stepper source in the host emulation, i.e. the F_FR instance, against the
oracle's mass matrix, bias forces and connect-equality rows.  The GPU twins are in tests/test_gpu_dynamics.py.

The emulation with a dynamics row is tests/emu/emu_dynamics.cpp (emu.cpp plus the row), built into its own library here.  The oracle side is an
oracle positioned at the same qpos / qvel and forward()ed: qM expanded with mj_fullM restated in numpy, qfrc_bias, the first 3 neq rows of efc_J /
efc_pos, and subtree_com for the reference's cassie_sim_centroid_inertia (src/cassiemujoco.c:1647-1687)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN
from test_frames import MODELS, ZERO_ROW, omodel
from test_model_variants import PD_ROW

COLS, M0, BIAS, JEQ, EQPOS, RCM = 40, 0, 1600, 1640, 2120, 2132
_LIB = None


def dyn_lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_dynamics.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_dynamics.cpp'), os.path.join(E.CSRC, 'mjcf.cpp'), os.path.join(E.HERE, 'emu', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], srcs[1]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_dyn_new.restype = vp
        L.emu_dyn_new.argtypes = [C.c_char_p, ci]
        L.emu_dyn_free.argtypes = [vp]
        L.emu_dyn_compute.argtypes = [vp, dp]
        L.emu_step.argtypes = [vp, dp, ci]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_model_set.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set_const.argtypes = [vp]
        _LIB = L
    return _LIB


class DynSim:
    """one emulated environment; dynamics() runs launch mode 5 of the F_ALL | F_FR source at the current state"""

    def __init__(self, model, fp32=False):
        self.L = dyn_lib()
        self.h = self.L.emu_dyn_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model
        assert self.L.emu_dyn_width() == 2144

    def close(self):
        if self.h:
            self.L.emu_dyn_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def step(self, pd50, nticks=1):
        a = np.ascontiguousarray(pd50, dtype=np.float64)
        self.L.emu_step(self.h, a.ctypes.data_as(C.POINTER(C.c_double)), nticks)

    def model_set(self, what, v):
        a = np.ascontiguousarray(v, dtype=np.float64)
        assert self.L.emu_model_set(self.h, what.encode(), a.ctypes.data_as(C.POINTER(C.c_double)), a.size) == 0, what

    def dynamics(self):
        out = np.zeros(2144)
        self.L.emu_dyn_compute(self.h, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out


def unpack(row, nv, neq):
    """the row's parts in the shapes of cassie_batch_get_dynamics"""
    M = row[M0:M0 + COLS * COLS].reshape(COLS, COLS)
    J = row[JEQ:JEQ + 12 * COLS].reshape(12, COLS)
    return dict(M=M[:nv, :nv], bias=row[BIAS:BIAS + nv], J_eq=J[:3 * neq, :nv], eq_err=row[EQPOS:EQPOS + 3 * neq], rcm=row[RCM:RCM + 3], full=M, Jfull=J)


def full_m(qM, m):
    """mj_fullM: the sparse qM (row i: i and its ancestors, from dof_Madr[i]) as a dense symmetric matrix"""
    madr, parent = m['dof_Madr'].astype(int), m['dof_parentid'].astype(int)
    nv = madr.size
    M = np.zeros((nv, nv))
    for i in range(nv):
        a, j = madr[i], i
        while j >= 0:
            M[i, j] = M[j, i] = qM[a]
            a += 1
            j = parent[j]
    return M


def centroid(M, rcm):
    """cassie_sim_centroid_inertia's formula, sign of the off-diagonals included"""
    m, Ip, r = M[0, 0], M[3:6, 3:6], rcm
    Ic = np.zeros((3, 3))
    Ic[0, 0] = Ip[0, 0] - m * (r[1] ** 2 + r[2] ** 2)
    Ic[1, 1] = Ip[1, 1] - m * (r[2] ** 2 + r[0] ** 2)
    Ic[2, 2] = Ip[2, 2] - m * (r[0] ** 2 + r[1] ** 2)
    Ic[0, 1] = Ic[1, 0] = Ip[1, 0] - m * r[1] * r[0]
    Ic[1, 2] = Ic[2, 1] = Ip[2, 1] - m * r[2] * r[1]
    Ic[2, 0] = Ic[0, 2] = Ip[2, 0] - m * r[2] * r[0]
    return Ic


def oracle_dynamics(O, model, qpos, qvel, consts=None):
    """the oracle at (qpos, qvel), forward()ed: dense M, qfrc_bias, the connect rows and their errors; then, as the reference's centroid_inertia
    does it, the pelvis quaternion set to identity and forward()ed again: M and subtree_com of the world body minus the pelvis position"""
    m = omodel(model)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    if consts:
        for k, v in consts.items():
            o.model_arr(k)[:] = v
        o.just_set_const()   # subtree masses (subtree_com) follow the new body masses, as the batch's set_const does for its constant row
    o.arr('qpos')[:] = qpos[:o.nq]
    o.arr('qvel')[:] = qvel[:o.nv]
    o.forward()
    neq = m['eq_obj1id'].size
    out = dict(M=full_m(o.arr('qM'), m), bias=o.arr('qfrc_bias').copy(), J_eq=o.efc_J()[:3 * neq].copy(), eq_err=o.arr('efc_pos')[:3 * neq].copy())
    q = o.arr('qpos')
    q[3:7] = [1, 0, 0, 0]
    o.forward()
    Mi = full_m(o.arr('qM'), m)
    out['rcm'] = o.arr('subtree_com')[0:3] - q[0:3]
    out['Icm'] = centroid(Mi, out['rcm'])
    o.close()
    return out


def states(e, model, nticks=600, every=60):
    """(qpos, qvel) of the emulation through a stance (first half) and a fall with the motors off, every `every` ticks"""
    nq = omodel(model)['qpos_spring'].size
    xb = model == 'cassie_tray_box'
    for k in range(nticks):
        e.step(PD_ROW if k < nticks // 2 else ZERO_ROW)
        if k % every == every - 1:
            qv = e.get('qvel')
            if xb:
                qv = np.concatenate([qv, e.get('xqvel')])
            yield k, e.get('qpos')[:nq], qv


def _compare(oracle_mod, model, fp32):
    e = DynSim(model, fp32=fp32)
    nv = 38 if model == 'cassie_tray_box' else 32
    neq = omodel(model)['eq_obj1id'].size
    err = dict(M=0.0, bias=0.0, J_eq=0.0, eq_err=0.0, rcm=0.0, Icm=0.0)
    scale = dict(M=0.0, bias=0.0, J_eq=0.0, eq_err=0.0, rcm=0.0, Icm=0.0)
    for k, q, v in states(e, model):
        got, want = unpack(e.dynamics(), nv, neq), oracle_dynamics(oracle_mod, model, q, v)
        got['Icm'] = centroid(got['M'], got['rcm'])
        for key in err:
            err[key] = max(err[key], np.abs(got[key] - want[key]).max())
            scale[key] = max(scale[key], np.abs(want[key]).max())
        assert not got['full'][nv:, :].any() and not got['full'][:, nv:].any() and not got['Jfull'][3 * neq:].any() and not got['Jfull'][:, nv:].any()
    e.close()
    return err, scale


# measured over the four models (host emulation): fp64 M <= 2.1e-16, bias <= 4.9e-16, J_eq <= 9.4e-16, Icm <= 6.1e-15 of their largest entries,
# eq_err <= 3.9e-16 m, rcm <= 8.5e-16 m; fp32 M, bias, J_eq <= 5.1e-7 and Icm <= 1.6e-6 of their largest entries, eq_err <= 2.0e-7 m, rcm <= 3.1e-7 m.
# The bars sit about an order of magnitude above these.
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box', 'cassie_mass', 'cassie_hfield'])
def test_dynamics_follow_the_oracle_fp64(oracle_mod, model):
    err, scale = _compare(oracle_mod, model, False)
    print(model, {k: err[k] / scale[k] for k in err}, err['eq_err'])
    assert err['M'] <= 1e-14 * scale['M'] and err['J_eq'] <= 1e-14 * scale['J_eq'], (err, scale)
    assert err['bias'] <= 1e-14 * scale['bias'] and err['eq_err'] <= 1e-14, (err, scale)
    assert err['rcm'] <= 1e-14 and err['Icm'] <= 1e-13 * scale['Icm'], (err, scale)


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box', 'cassie_mass', 'cassie_hfield'])
def test_dynamics_follow_the_oracle_fp32(oracle_mod, model):
    err, scale = _compare(oracle_mod, model, True)
    print(model, {k: err[k] / scale[k] for k in err}, err['eq_err'])
    for key in ('M', 'bias', 'J_eq', 'Icm'):
        assert err[key] <= 1e-5 * scale[key], (key, err, scale)
    assert err['eq_err'] <= 2e-6 and err['rcm'] <= 3e-6, (err, scale)


def test_dynamics_with_per_environment_constants(oracle_mod):
    """body_mass / body_ipos / dof_damping of the env's constant row (domain randomisation): M and bias follow an oracle given those constants"""
    m = omodel('cassie')
    rng = np.random.default_rng(3)
    mass = m['body_mass'] * rng.uniform(0.8, 1.2, m['body_mass'].size)
    ipos = m['body_ipos'] + rng.uniform(-0.01, 0.01, m['body_ipos'].size)
    damp = m['dof_damping'] * rng.uniform(0.5, 1.5, m['dof_damping'].size)
    e = DynSim('cassie')
    e.model_set('body_mass', mass)
    e.model_set('body_ipos', ipos)
    e.model_set('dof_damping', damp)
    e.L.emu_set_const(e.h)
    worst = dict(M=0.0, bias=0.0, rcm=0.0)
    for k, q, v in states(e, 'cassie', nticks=300, every=100):
        got = unpack(e.dynamics(), 32, 4)
        want = oracle_dynamics(oracle_mod, 'cassie', q, v, dict(body_mass=mass, body_ipos=ipos, dof_damping=damp))
        for key in worst:
            worst[key] = max(worst[key], np.abs(got[key] - want[key]).max() / max(1e-300, np.abs(want[key]).max()))
        plain = oracle_dynamics(oracle_mod, 'cassie', q, v)
        assert np.abs(plain['M'] - want['M']).max() > 1e-3   # the constants matter
    print(worst)
    assert worst['M'] <= 1e-12 and worst['bias'] <= 1e-10 and worst['rcm'] <= 1e-12, worst


@pytest.mark.parametrize('fp32', [False, True])
def test_dynamics_launch_writes_nothing_else(fp32):
    """mode 5 changes no state array: bitwise, right after each call and in the steps that follow, against a twin that never asked"""
    a, b = DynSim('cassie', fp32=fp32), DynSim('cassie', fp32=fp32)
    fields = ('qpos', 'qvel', 'qacc_ws', 'obs', 'aux', 'counters', 'cst', 'dfilt', 'xfrc')
    for k in range(400):
        row = PD_ROW if k < 200 else ZERO_ROW
        a.step(row)
        b.step(row)
        if k % 10 == 0:
            before = {f: b.get(f) for f in fields}
            b.dynamics()
            for f in fields:
                assert np.array_equal(before[f], b.get(f)), (k, f)
                assert np.array_equal(a.get(f), b.get(f)), (k, f)
    for f in fields:
        assert np.array_equal(a.get(f), b.get(f)), f


def test_dynamics_row_is_symmetric_and_positive():
    e = DynSim('cassie')
    for k, q, v in states(e, 'cassie', nticks=200, every=100):
        M = unpack(e.dynamics(), 32, 4)['M']
        assert np.array_equal(M, M.T)
        assert np.linalg.eigvalsh(M).min() > 0


def test_achilles_connects_are_equalities_1_and_3():
    """cassie_sim_loop_constraint_info picks the connects whose body1 is left- / right-achilles-rod: equalities 1 and 3 of cassie, the ones the
    reference finds by the names left- / right-achilles-rod-eq"""
    for model in ('cassie', 'cassie_tray_box', 'cassie_mass', 'cassie_hfield'):
        m = omodel(model)
        names = list(m['names_body'])
        picked = [e for e, b in enumerate(m['eq_obj1id'].astype(int)) if names[b] in ('left-achilles-rod', 'right-achilles-rod')]
        assert picked == [1, 3], (model, picked)
