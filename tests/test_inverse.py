"""Inverse rows (cassie_batch_inverse, launch mode 6): mj_inverse of MuJoCo 2.1.0 at a caller's qacc.  The restatement on the fp64 oracle
(tests/inverse_support.py) is pinned by the forward / inverse round trip, and the product's stepper source in the host emulation, i.e. the F_FR instances,
follows it.  The GPU twins are in tests/test_gpu_inverse.py.

The emulation with an inverse row is tests/emu/emu_inverse.cpp (emu_env_contact.cpp plus the row), built into its own library here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from contact_support import random_contact
from inverse_support import WIDTH, columns, inverse, oracle_at, scale, unpack
from mechanics_support import random_mechanics, table
from test_env_body_pos import offsets
from test_frames import MODELS, ZERO_ROW
from test_hfield import terrain
from test_model_variants import PD_ROW

MODELS_CHECKED = ['cassie', 'cassie_tray_box', 'cassie_hfield']
MC_INERTIA, MC_ARMATURE, MC_STIFF, MC_SPRING, MECH_W, BP_W = 0, 96, 128, 160, 192, 96
_LIB = None


def inv_lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_inverse.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_inverse.cpp'), os.path.join(E.CSRC, 'mjcf.cpp'), os.path.join(E.HERE, 'emu', 'emu.cpp'),
                os.path.join(E.HERE, 'emu', 'emu_env_contact.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], srcs[1]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_ct_new.restype = vp
        L.emu_ct_new.argtypes = [C.c_char_p, ci]
        L.emu_inv_free.argtypes = [vp]
        L.emu_inv_compute.argtypes = [vp, dp, dp]
        L.emu_inv_set_rows.argtypes = [vp, dp, dp]
        L.emu_ct_mode.argtypes = [vp, ci]
        L.emu_ct_set.argtypes = [vp, dp, dp, dp]
        L.emu_ct_step.argtypes = [vp, dp, ci]
        L.emu_set_hfield.argtypes = [vp, C.POINTER(C.c_float), ci]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class InvSim:
    """one emulated environment; inverse(qacc) runs launch mode 6 of the F_FR source at the current state"""

    def __init__(self, model, fp32=False, hfield=None):
        self.L = inv_lib()
        self.model, self.nv = model, 38 if model == 'cassie_tray_box' else 32
        self.h = self.L.emu_ct_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model
        assert self.L.emu_inv_width() == WIDTH
        if hfield is not None:
            self.L.emu_set_hfield(self.h, hfield.ctypes.data_as(C.POINTER(C.c_float)), hfield.size)

    def close(self):
        if self.h:
            self.L.emu_inv_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), _dp(buf), n)
        assert k >= 0, name
        return buf[:k]

    def state(self):
        q = self.get('qpos')
        v = self.get('qvel')
        if self.nv == 38:
            v = np.concatenate([v, self.get('xqvel')])
        return q, v

    def step(self, pd50, nticks=1):
        a = np.ascontiguousarray(pd50, dtype=np.float64)
        self.L.emu_ct_step(self.h, _dp(a), nticks)

    def env_rows(self, mech=None, body_pos=None, contact=None):
        """step and invert with this environment's own rows (the F_BP | F_AC | F_MC | F_CT source): mechanics (inertia, armature, stiffness,
        springref) as mechanics_support gives them, body_pos [nbody, 3], contact (solref, solimp, solmix) per geom"""
        t = table(self.model)
        self.L.emu_ct_mode(self.h, 2)
        mrow = brow = None
        if mech is not None:
            I, arm, k, q = mech
            mrow = np.zeros(MECH_W)
            mrow[MC_INERTIA:MC_INERTIA + I.size] = I.ravel()
            for d in range(32):
                j = int(t['dof_jntid'][d])
                mrow[MC_ARMATURE + d], mrow[MC_STIFF + d], mrow[MC_SPRING + d] = arm[d], k[j], q[j]
        if body_pos is not None:
            brow = np.zeros(BP_W)
            brow[:body_pos.size] = body_pos.ravel()
        self.L.emu_inv_set_rows(self.h, _dp(brow) if brow is not None else None, _dp(mrow) if mrow is not None else None)
        if contact is not None:
            sr, si, sm = [np.ascontiguousarray(x, dtype=np.float64) for x in contact]
            self.L.emu_ct_set(self.h, _dp(sr), _dp(si), _dp(sm))

    def inverse(self, qacc):
        a, out = np.ascontiguousarray(columns(qacc, self.nv)), np.zeros(WIDTH)
        self.L.emu_inv_compute(self.h, _dp(a), _dp(out))
        return out


def gait_row(k):
    """the standing PD row with its targets swung: a stepping-like motion with feet leaving and striking the ground"""
    row = PD_ROW.copy()
    s = np.sin(2 * np.pi * 1.5 * k * 5e-4)
    row[10 + 2], row[15 + 2] = row[10 + 2] + 0.35 * s, row[15 + 2] - 0.35 * s
    row[10 + 3], row[15 + 3] = row[10 + 3] - 0.3 * max(s, 0), row[15 + 3] - 0.3 * max(-s, 0)
    return row


def phases(e, nticks=900, every=75):
    """(tick, phase, qpos, qvel) of the emulation through a stance, a gait and a fall with the motors off"""
    for k in range(nticks):
        ph = 'stance' if k < nticks // 3 else ('gait' if k < 2 * nticks // 3 else 'fall')
        e.step(PD_ROW if ph == 'stance' else (gait_row(k) if ph == 'gait' else ZERO_ROW))
        if k % every == every - 1:
            q, v = e.state()
            yield k, ph, q, v


def qacc_kinds(o, nv, rng):
    """the three qacc of every check: the oracle's solved qacc at the state (zero ctrl), zero, and the solved one plus a seeded perturbation"""
    solved = o.arr('qacc')[:nv].copy()
    return dict(solved=solved, zero=np.zeros(nv), perturbed=solved + rng.normal(0, 1, nv) * (1 + np.abs(solved)) * 0.3)


def _compare(O, model, fp32, rows=None, seed=0):
    """errors of the emulation against the restatement, per sample relative to inverse_support.scale; the inequality-row activity seen"""
    hf = terrain(7) if model == 'cassie_hfield' else None
    e = InvSim(model, fp32=fp32, hfield=hf)
    lines = {}
    if rows:
        e.env_rows(**rows)
        if 'mech' in rows:
            lines.update(zip(('inertia', 'armature', 'stiffness', 'springref'), rows['mech']))
        if 'body_pos' in rows:
            lines['body_pos'] = rows['body_pos']
        if 'contact' in rows:
            lines.update(geom_solref=rows['contact'][0], geom_solimp=rows['contact'][1], geom_solmix=rows['contact'][2])
    rng = np.random.default_rng(seed)
    err = dict(qfrc_inverse=[], qfrc_constraint=[])
    active = inactive = 0
    for k, ph, q, v in phases(e):
        o = oracle_at(O, model, q, v, hfield=hf, **lines)
        for kind, qa in qacc_kinds(o, e.nv, rng).items():
            want, got = inverse(o, model, qa), unpack(e.inverse(qa), e.nv)
            assert (got['nefc'], got['ncon']) == (want['nefc'], want['ncon']), (model, k, kind, got['nefc'], want['nefc'], got['ncon'], want['ncon'])
            for key in err:
                err[key].append(np.abs(got[key] - want[key]).max() / scale(want))
            active += int((want['f'][want['ineq']] > 0).sum())
            inactive += int((want['f'][want['ineq']] == 0).sum())
        o.close()
    e.close()
    return {k: np.array(v) for k, v in err.items()}, active, inactive


# ------------------------------------------------------------------ 1. the restatement closes the forward / inverse round trip on the oracle
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box', 'cassie_hfield'])
def test_round_trip_closes_on_the_oracle(oracle_mod, model):
    """a converged forward (iterations 10 000, tolerance 0) with PD-like torques, xfrc_applied and qfrc_applied; the inverse at its solved qacc gives back
    qfrc_actuator + qfrc_applied + sum J(xipos)' xfrc = qfrc_smooth - qfrc_passive + qfrc_bias, and the forward's own qfrc_constraint"""
    hf = terrain(7) if model == 'cassie_hfield' else None
    e = InvSim(model, hfield=hf)
    rng = np.random.default_rng(11)
    worst = dict(tight=0.0, loose=0.0, qc=0.0)
    for k, ph, q, v in phases(e, nticks=600, every=100):
        for label, lines in (('tight', dict(opt_iterations=[10000], opt_tolerance=[0.0])), ('loose', {})):
            o = oracle_at(oracle_mod, model, q, v, hfield=hf, **lines)
            o.arr('ctrl')[:] = rng.uniform(-20, 20, o.arr('ctrl').size)
            x = o.arr('xfrc_applied').reshape(-1, 6)
            x[1:] = rng.normal(0, 5, x[1:].shape)
            o.arr('qfrc_applied')[:] = rng.normal(0, 3, o.nv)
            o.forward()
            want = o.arr('qfrc_smooth') - o.arr('qfrc_passive') + o.arr('qfrc_bias')
            got = inverse(o, model, o.arr('qacc').copy())
            scale = np.abs(want).max()
            worst[label] = max(worst[label], np.abs(got['qfrc_inverse'] - want).max() / scale)
            if label == 'tight':
                worst['qc'] = max(worst['qc'], np.abs(got['qfrc_constraint'] - o.arr('qfrc_constraint')).max() / scale)
            o.close()
    e.close()
    print(model, worst)
    assert worst['tight'] <= 1e-8 and worst['qc'] <= 1e-8, worst
    assert worst['loose'] <= 1e-2, worst   # 50 iterations, tolerance 1e-8: the solver's own accuracy


def test_restatement_matches_mujoco_rules(oracle_mod):
    """equality rows always carry -jar / R, inequality rows only when jar < 0; at qacc = 0 a standing robot's contacts push (f > 0)"""
    e = InvSim('cassie')
    for _ in range(300):
        e.step(PD_ROW)
    q, v = e.state()
    o = oracle_at(oracle_mod, 'cassie', q, v)
    r = inverse(o, 'cassie', np.zeros(32))
    eq = ~r['ineq']
    assert np.allclose(r['f'][eq], -r['jar'][eq] * o.arr('efc_D')[eq], rtol=0, atol=0)
    assert (r['f'][r['ineq']] >= 0).all() and (r['f'][r['ineq'] & (r['jar'] >= 0)] == 0).all()
    assert r['ncon'] >= 2 and (r['f'][r['ineq']] > 0).sum() >= 4
    o.close()
    e.close()


# ------------------------------------------------------------------ 2. the emulated F_FR source follows the restatement
@pytest.mark.parametrize('model', MODELS_CHECKED)
def test_inverse_follows_the_oracle_fp64(oracle_mod, model):
    err, active, inactive = _compare(oracle_mod, model, False)
    print(model, {k: (v.max(), np.median(v)) for k, v in err.items()}, active, inactive)
    assert active > 0 and inactive > 0, (active, inactive)
    assert err['qfrc_inverse'].max() <= 1e-10 and err['qfrc_constraint'].max() <= 1e-10, err


# measured in the host emulation, of the largest term (inverse_support.scale), over the 36 samples of each model: fp64 <= 5.7e-13 (cassie 4.1e-13,
# cassie_tray_box 5.7e-13, cassie_hfield 1.6e-13; with per-environment rows <= 2.9e-13); fp32 worst / 90th percentile / median: cassie 3.5e-4 / 2.6e-4 /
# 9.0e-5, cassie_tray_box 8.1e-4 / 4.4e-4 / 2.3e-5, cassie_hfield 1.7e-4 / 1.1e-4 / 1.3e-5 (DESIGN.md section 3).  The bars sit about 4x above the worst.
FP32_BARS = dict(qfrc_inverse=3e-3, qfrc_constraint=3e-3)


@pytest.mark.parametrize('model', MODELS_CHECKED)
def test_inverse_follows_the_oracle_fp32(oracle_mod, model):
    err, active, inactive = _compare(oracle_mod, model, True)
    print(model, {k: (v.max(), np.percentile(v, 90), np.median(v)) for k, v in err.items()})
    for key, bar in FP32_BARS.items():
        assert err[key].max() <= bar, (key, err[key].max())


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_inverse_with_per_environment_rows(oracle_mod, model):
    """this environment's mechanics, body offsets and contact softness, against an oracle given the same tables"""
    rows = dict(mech=random_mechanics(model, 5), body_pos=offsets(model, 5), contact=random_contact(model, 5))
    err, active, inactive = _compare(oracle_mod, model, False, rows=rows, seed=1)
    print(model, {k: v.max() for k, v in err.items()}, active, inactive)
    assert active > 0 and err['qfrc_inverse'].max() <= 1e-10 and err['qfrc_constraint'].max() <= 1e-10, err


# ------------------------------------------------------------------ 3. mode 6 writes nothing else
@pytest.mark.parametrize('fp32', [False, True])
def test_inverse_launch_writes_nothing_else(fp32):
    """state, warm start, observations, aux, counters and controller rows bitwise unchanged right after each call, and in the steps that follow,
    against a twin that never asked"""
    a, b = InvSim('cassie_tray_box', fp32=fp32), InvSim('cassie_tray_box', fp32=fp32)
    fields = ('qpos', 'qvel', 'xqvel', 'qacc_ws', 'obs', 'aux', 'counters', 'cst', 'dfilt', 'xfrc')
    rng = np.random.default_rng(2)
    for k in range(400):
        row = PD_ROW if k < 200 else ZERO_ROW
        a.step(row)
        b.step(row)
        if k % 10 == 0:
            before = {f: b.get(f) for f in fields}
            b.inverse(rng.normal(0, 5, 38))
            for f in fields:
                assert np.array_equal(before[f], b.get(f)), (k, f)
                assert np.array_equal(a.get(f), b.get(f)), (k, f)
    for f in fields:
        assert np.array_equal(a.get(f), b.get(f)), f
    a.close()
    b.close()


def test_holding_torques_carry_the_weight():
    """qacc = 0 once the robot has settled on its PD stand (2 s; it rocks onto three contacts first): the unactuated pelvis dofs need (almost)
    nothing once the ground's forces are in, unlike M qacc + bias - passive"""
    e = InvSim('cassie')
    e.step(PD_ROW, 4000)
    got = unpack(e.inverse(np.zeros(32)), 32)
    pelvis_z = got['qfrc_inverse'][2]
    without = got['qfrc_inverse'][2] + got['qfrc_constraint'][2]
    assert without > 200 and abs(pelvis_z) < 0.02 * without and np.abs(got['qfrc_inverse'][:6]).max() < 0.02 * without, (got['qfrc_inverse'][:6], without)
    assert got['ncon'] >= 2 and got['dropped'] == 0
    e.close()
