"""Acceleration rows (cassie_batch_enable_accelerations): the product's stepper source in the host emulation with a frame table and an acceleration row,
i.e. the F_FR instance and the kernel wrapper's accel_row, against the oracle.  The GPU twins are in tests/test_gpu_accelerations.py.

The emulation is tests/emu/emu_accel.cpp (emu.cpp plus the rows), built into its own library here.  The oracle side restates the reference queries:
cassie_sim_qacc returns d->qacc (src/cassiemujoco.c:1216-1219); cassie_sim_body_acceleration (:1762-1771) runs mj_comVel and mj_rnePostConstraint on
mjData as the step left it -- the new qvel, the cdof of the state the last sub-step started from, the last qacc -- and copies cacc.  The numpy
restatement of those two functions is checked against the oracle's own cdof_dot / cvel / cacc first, on arrays where the oracle computed them itself."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from test_frames import all_frames, omodel
from test_model_variants import PD_ROW

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
ZERO_ROW = np.zeros(50)   # no torque, no gains: the robot falls
QCOLS, SLOT, FRAME_W = 40, 8, 20
JNT_FREE, JNT_BALL = 0, 1
_LIB = None


def ac_lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_accel.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_accel.cpp'), os.path.join(E.CSRC, 'mjcf.cpp'), os.path.join(E.HERE, 'emu', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], srcs[1]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_ac_new.restype = vp
        L.emu_ac_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_ac_free', 'emu_ac_forward', 'emu_plain'):
            getattr(L, n).argtypes = [vp]
        L.emu_ac_set_frames.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(ci), ci]
        L.emu_ac_enable.argtypes = [vp, ci]
        L.emu_ac_step.argtypes = [vp, dp, ci]
        for n in ('emu_ac_row', 'emu_ac_frames', 'emu_ac_get_xws', 'emu_ac_set_xws'):
            getattr(L, n).argtypes = [vp, dp]
        L.emu_ac_width.argtypes = [ci]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class AccSim:
    """one emulated environment on the extended instance; with frames or the acceleration row on, the F_FR path and accel_row run"""

    def __init__(self, model, fp32=False):
        self.L = ac_lib()
        self.h = self.L.emu_ac_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model

    def close(self):
        if self.h:
            self.L.emu_ac_free(self.h)
            self.h = None

    def set_frames(self, names, kinds):
        arr = (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])
        ks = (C.c_int * max(1, len(kinds)))(*kinds)
        return self.L.emu_ac_set_frames(self.h, arr, ks, len(names))

    def enable(self, on=True):
        self.L.emu_ac_enable(self.h, 1 if on else 0)

    def row(self):
        buf = np.zeros(QCOLS + SLOT * 64)
        n = self.L.emu_ac_row(self.h, _dp(buf))
        return None if n < 0 else buf[:n]

    def frames(self):
        buf = np.zeros(64 * FRAME_W)
        n = self.L.emu_ac_frames(self.h, _dp(buf))
        return buf[:n * FRAME_W]

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), _dp(buf), n)
        assert k >= 0, name
        return buf[:k]

    def set(self, name, values):
        a = np.ascontiguousarray(values, dtype=np.float64)
        assert self.L.emu_set(self.h, name.encode(), _dp(a), a.size) >= 0, name

    def xws(self):
        buf = np.zeros(6)
        self.L.emu_ac_get_xws(self.h, _dp(buf))
        return buf

    def set_xws(self, values):
        self.L.emu_ac_set_xws(self.h, _dp(np.ascontiguousarray(values, dtype=np.float64)))

    def step(self, pd50, nticks=1):
        self.L.emu_ac_step(self.h, _dp(np.ascontiguousarray(pd50, dtype=np.float64)), nticks)

    def forward(self):
        self.L.emu_ac_forward(self.h)


# ---------------------------------------------------------------- the restatement of mj_comVel + mj_rnePostConstraint
def cross_motion(v, u):
    """mju_crossMotion: [w x u_ang; w x u_lin + v x u_ang]"""
    return np.r_[np.cross(v[:3], u[:3]), np.cross(v[:3], u[3:]) + np.cross(v[3:], u[:3])]


def restate(m, cdof, qvel, qacc):
    """(cvel [nbody, 6], cdof_dot [nv, 6], cacc [nbody, 6]) of mj_comVel + mj_rnePostConstraint from cdof, qvel and qacc: per body, the joint-type rules
    of mj_comVel (free: translations 0, rotations from the cvel after the translations; ball: all three dofs from the cvel before the ball; hinge /
    slide: sequential), then cacc = cacc[parent] + sum cdof_dot qvel + cdof qacc with cacc[world] = (0, 0, 0, -g)"""
    parent, dofadr, dofnum = (m[k].astype(int) for k in ('body_parentid', 'body_dofadr', 'body_dofnum'))
    jtype, djnt = m['jnt_type'].astype(int), m['dof_jntid'].astype(int)
    nb, nv = parent.size, qvel.size
    cdof = cdof.reshape(nv, 6)
    cvel, cdd, cacc = np.zeros((nb, 6)), np.zeros((nv, 6)), np.zeros((nb, 6))
    cacc[0, 3:] = -m['opt_gravity']
    for i in range(1, nb):
        cv, bda, j = cvel[parent[i]].copy(), dofadr[i], 0
        while j < dofnum[i]:
            jt = jtype[djnt[bda + j]]
            if jt == JNT_FREE:
                for k in range(3):
                    cv = cv + cdof[bda + j + k] * qvel[bda + j + k]
                j += 3
                jt = JNT_BALL
            if jt == JNT_BALL:
                for k in range(3):
                    cdd[bda + j + k] = cross_motion(cv, cdof[bda + j + k])
                for k in range(3):
                    cv = cv + cdof[bda + j + k] * qvel[bda + j + k]
                j += 3
            else:
                cdd[bda + j] = cross_motion(cv, cdof[bda + j])
                cv = cv + cdof[bda + j] * qvel[bda + j]
                j += 1
        cvel[i] = cv
        a = cacc[parent[i]].copy()
        for j in range(dofnum[i]):
            a += cdd[bda + j] * qvel[bda + j] + cdof[bda + j] * qacc[bda + j]
        cacc[i] = a
    return cvel, cdd, cacc


def oracle_row(o, m, names, kinds):
    """the acceleration row the reference's queries give after the oracle's last step / forward: qacc, then per frame the restated cacc (sites 0)"""
    nv = o.nv
    _, _, cacc = restate(m, o.arr('cdof'), o.arr('qvel').copy(), o.arr('qacc').copy())
    row = np.zeros(QCOLS + SLOT * len(names))
    row[:nv] = o.arr('qacc')
    bodies = list(m['names_body'])
    for f, (name, kind) in enumerate(zip(names, kinds)):
        if kind == 0:
            row[QCOLS + SLOT * f:QCOLS + SLOT * f + 6] = cacc[bodies.index(name)]
    return row


def split(row, nframes):
    """(qacc [40], cacc [nframes, 6], pads [nframes, 2]) of an acceleration row"""
    s = row[QCOLS:QCOLS + SLOT * nframes].reshape(nframes, SLOT)
    return row[:QCOLS], s[:, :6], s[:, 6:]


MODELS_CHECKED = ['cassie', 'cassie_tray_box', 'cassie_hfield', 'cassie_no_grav']


@pytest.mark.parametrize('model', MODELS_CHECKED)
def test_restatement_reproduces_the_oracle(oracle_mod, model):
    """on the oracle's pre-Euler arrays (after a forward: cdof, qvel and qacc of one state) the restatement gives the oracle's own cvel, cdof_dot and
    cacc within 1e-12, through a stance and a fall"""
    O = oracle_mod
    m = omodel(model)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    stance, fall = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    worst, scale = 0.0, 0.0
    for k in range(600):
        o.step_pd(stance if k < 300 else fall)
        if k % 50 == 49:
            o.forward()
            cvel, cdd, cacc = restate(m, o.arr('cdof'), o.arr('qvel').copy(), o.arr('qacc').copy())
            for got, key in ((cvel, 'cvel'), (cdd, 'cdof_dot'), (cacc, 'cacc')):
                want = o.arr(key).reshape(got.shape)
                worst = max(worst, np.abs(got - want).max())
                scale = max(scale, np.abs(want).max())
    print(model, worst, scale)
    assert worst <= 1e-12 * max(1.0, scale) and scale > 1


def _frames(model):
    names, kinds = all_frames(model)
    return names, kinds


def _compare_steps(O, model, fp32=False, nticks=600, every=25):
    """stance for half the ticks, then a fall; the emulated acceleration row against the restated oracle every `every` ticks.  Returns the worst
    differences and the largest magnitudes of qacc and cacc, and the largest pad entry"""
    m = omodel(model)
    names, kinds = _frames(model)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    e = AccSim(model, fp32=fp32)
    e.enable(True)
    assert e.set_frames(names, kinds) == 0
    e.forward()
    stance, fall = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    worst, scale, pad = dict(qacc=0.0, cacc=0.0), dict(qacc=0.0, cacc=0.0), 0.0
    for k in range(nticks):
        u, row = (stance, PD_ROW) if k < nticks // 2 else (fall, ZERO_ROW)
        o.step_pd(u)
        e.step(row)
        if k % every == every - 1:
            gq, gc, gp = split(e.row(), len(names))
            wq, wc, _ = split(oracle_row(o, m, names, kinds), len(names))
            worst['qacc'] = max(worst['qacc'], np.abs(gq - wq).max())
            worst['cacc'] = max(worst['cacc'], np.abs(gc - wc).max())
            scale['qacc'] = max(scale['qacc'], np.abs(wq).max())
            scale['cacc'] = max(scale['cacc'], np.abs(wc).max())
            pad = max(pad, np.abs(gp).max())
    e.close()
    return worst, scale, pad


@pytest.mark.parametrize('model', MODELS_CHECKED)
def test_accelerations_follow_the_oracle_fp64(oracle_mod, model):
    worst, scale, pad = _compare_steps(oracle_mod, model)
    print(model, worst, scale)
    assert worst['qacc'] <= 1e-8 * scale['qacc'] and worst['cacc'] <= 1e-8 * scale['cacc'], (worst, scale)
    assert pad == 0 and scale['qacc'] > 1 and scale['cacc'] > 1


def _placed_forward(O, model, fp32, q, v, ws):
    """a fresh oracle and a fresh emulated environment placed at one state (qpos, qvel, warm start; zero ctrl), one forward each: (emulated row,
    oracle row, emulated warm start before and after)"""
    m = omodel(model)
    names, kinds = _frames(model)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    o.arr('qpos')[:] = q
    o.arr('qvel')[:] = v
    o.arr('qacc_warmstart')[:] = ws
    o.forward()
    e = AccSim(model, fp32=fp32)
    e.enable(True)
    assert e.set_frames(names, kinds) == 0
    nq = o.nq
    e.set('qpos', np.r_[q, np.zeros(44 - nq)])
    e.set('qvel', v[:32])
    e.set('qacc_ws', ws[:32])
    if o.nv > 32:
        e.set('xqvel', v[32:])
        e.set_xws(ws[32:])
    before = np.r_[e.get('qacc_ws')[:32], e.xws()]
    e.forward()
    after = np.r_[e.get('qacc_ws')[:32], e.xws()]
    got, want = e.row(), oracle_row(o, m, names, kinds)
    e.close()
    o.close()
    return got, want, before, after, len(names)


def _oracle_states(O, model, ticks=600, every=100):
    """(qpos, qvel, qacc_warmstart) of the oracle through a stance and a fall"""
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    stance, fall = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    out = []
    for k in range(ticks):
        o.step_pd(stance if k < ticks // 2 else fall)
        if k % every == every - 1:
            out.append((o.arr('qpos').copy(), o.arr('qvel').copy(), o.arr('qacc_warmstart').copy()))
    o.close()
    return out


@pytest.mark.parametrize('model', MODELS_CHECKED)
@pytest.mark.parametrize('fp32', [False, True])
def test_forward_at_the_oracle_state(oracle_mod, model, fp32):
    """mode 1 placed at oracle states of a stance and a fall: qacc is the oracle's forward qacc and cacc its restated query, and the warm start is left
    as it was.  fp64: within 1e-8 of the largest magnitude compared (of 1 where everything is smaller: cassie_no_grav floats nearly at rest).  fp32: the
    single-precision solve of the stiff closed-chain rows carries an absolute error of up to ~0.5 m/s^2 at these states (1.8e-3 of the largest
    magnitude at worst), so the bar is 1e-2 of the largest magnitude, or of 20 m/s^2 where everything is smaller"""
    bar, floor = (1e-2, 20.0) if fp32 else (1e-8, 1.0)
    for q, v, ws in _oracle_states(oracle_mod, model):
        got, want, before, after, nf = _placed_forward(oracle_mod, model, fp32, q, v, ws)
        gq, gc, _ = split(got, nf)
        wq, wc, _ = split(want, nf)
        assert np.abs(gq - wq).max() <= bar * max(floor, np.abs(wq).max()), (np.abs(gq - wq).max(), np.abs(wq).max())
        assert np.abs(gc - wc).max() <= bar * max(floor, np.abs(wc).max()), (np.abs(gc - wc).max(), np.abs(wc).max())
        assert np.array_equal(before, after)


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
@pytest.mark.parametrize('fp32', [False, True])
def test_step_qacc_is_the_warm_start_bitwise(model, fp32):
    """after a step the qacc part is, bit for bit, the warm start the step kept (the extra free body's too); beyond nv it reads zero"""
    names, kinds = _frames(model)
    e = AccSim(model, fp32=fp32)
    e.enable(True)
    assert e.set_frames(names, kinds) == 0
    e.forward()
    nv = 38 if model == 'cassie_tray_box' else 32
    for k in range(300):
        e.step(PD_ROW if k < 150 else ZERO_ROW)
        if k % 10 == 9:
            q = e.row()[:QCOLS]
            ws = e.get('qacc_ws')[:32]
            assert np.array_equal(q[:32], ws), k
            if nv > 32:
                assert np.array_equal(q[32:38], e.xws()), k
            assert not q[nv:].any()
    e.close()


@pytest.mark.parametrize('frames', [True, False])
@pytest.mark.parametrize('fp32', [False, True])
def test_accelerations_change_nothing_else(frames, fp32):
    """with the acceleration row on, qpos, qvel, obs, aux, the frame rows and the counters are bitwise those of a twin without it (with frames: both
    run the F_FR path; without: the twin runs the shipped extended instance)"""
    a, b = AccSim('cassie_tray_box', fp32=fp32), AccSim('cassie_tray_box', fp32=fp32)
    names, kinds = _frames('cassie_tray_box')
    if frames:
        assert a.set_frames(names, kinds) == 0 and b.set_frames(names, kinds) == 0
    b.enable(True)
    a.forward()
    b.forward()
    for k in range(400):
        row = PD_ROW if k < 200 else ZERO_ROW
        a.step(row)
        b.step(row)
        if k % 20 == 19:
            for f in ('qpos', 'qvel', 'xqvel', 'qacc_ws', 'obs', 'aux', 'counters', 'cst'):
                assert np.array_equal(a.get(f), b.get(f)), (k, f)
            assert np.array_equal(a.xws(), b.xws()) and np.array_equal(a.frames(), b.frames()), k
    assert np.abs(b.row()[:QCOLS]).max() > 1
    a.close()
    b.close()


def test_row_edge_cases():
    """no row before enable and after enable(0); the row follows set_frames to 40 + 8 count, zero until the next launch; acceleration rows without
    frames carry qacc only; the world reads (0, 0, 0, -g), a site zero, a body without dofs its parent's cacc"""
    e = AccSim('cassie')
    assert e.row() is None
    e.enable(True)
    assert e.row().size == 40 and not e.row().any()
    e.forward()
    assert e.row().size == 40 and np.abs(e.row()).max() > 1
    assert e.set_frames(['world', 'cassie-pelvis', 'left-toe', 'left-foot'], [0, 0, 1, 0]) == 0
    assert e.row().size == 40 + 8 * 4 and not e.row().any()
    assert ac_lib().emu_ac_width(4) == 72
    e.step(PD_ROW)
    q, c, _ = split(e.row(), 4)
    assert np.array_equal(c[0], [0, 0, 0, 0, 0, 9.81]) and not c[2].any() and np.abs(c[1]).max() > 0
    assert e.set_frames(['no-such-body'], [0]) == -1 and e.row().size == 72   # a refused table changes nothing
    e.enable(False)
    assert e.row() is None
    e.step(PD_ROW)
    e.close()


def test_dofless_body_reads_its_parent():
    """a body without dofs (the tray box's tray, welded to the pelvis side of the tree) carries its parent's cacc bitwise"""
    m = omodel('cassie_tray_box')
    dofnum, parent = m['body_dofnum'].astype(int), m['body_parentid'].astype(int)
    names = list(m['names_body'])
    dofless = [b for b in range(1, len(names)) if dofnum[b] == 0 and parent[b] > 0]
    assert dofless
    b = dofless[0]
    e = AccSim('cassie_tray_box')
    e.enable(True)
    assert e.set_frames([names[b], names[parent[b]]], [0, 0]) == 0
    e.forward()
    for _ in range(50):
        e.step(PD_ROW)
    _, c, _ = split(e.row(), 2)
    assert np.array_equal(c[0], c[1]) and np.abs(c[0]).max() > 0
    e.close()


def test_header_constants():
    """include/cassie_b200.h's CASSIE_ACC_* layout is the emulated row's"""
    txt = open(os.path.join(REPO, 'include', 'cassie_b200.h')).read()
    for name, value in (('CASSIE_ACC_QACC', 0), ('CASSIE_ACC_QCOLS', QCOLS), ('CASSIE_ACC_CACC', QCOLS), ('CASSIE_ACC_SLOT', SLOT)):
        assert '#define %s %d\n' % (name, value) in txt, name
    assert '#define CASSIE_ACC_WIDTH(count) (40 + 8 * (count))' in txt
