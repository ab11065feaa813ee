"""Per-tick traces (cassie_batch_set_trace): the product's stepper source in the host emulation with a trace row, i.e. the F_TC instances, against
the rows one-tick launches leave, the chain twin it is the twin of, and the fp64 oracle tick by tick.  The GPU twins are in tests/test_gpu_trace.py.

The emulation is tests/emu/emu_trace.cpp, built into its own library here: the trace twin's source with model-valued offset, actuator, mechanics and
contact rows, zero applied forces, a frame table and the trace row; or the chain twin's source on the same rows."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from test_frames import all_frames

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
ZERO_ROW = np.zeros(50)   # no torque, no gains: the robot falls
QPOS, QVEL, OBS, AUX, FRAME = range(5)   # include/cassie_b200.h CASSIE_TRACE_*
OBS_W, AUX_W, FRAME_W = 112, 64, 20
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_trace.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_trace.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci, ip = C.c_void_p, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int)
        L.emu_tc_new.restype = vp
        L.emu_tc_new.argtypes = [C.c_char_p, ci]
        L.emu_tc_free.argtypes = [vp]
        L.emu_tc_forward.argtypes = [vp]
        L.emu_tc_set_frames.argtypes = [vp, C.POINTER(C.c_char_p), ip, ci]
        L.emu_tc_set_trace.argtypes = [vp, ip, ip, ci, ci]
        L.emu_tc_traced.argtypes = [vp, ci]
        L.emu_tc_step.argtypes = [vp, dp, ci]
        L.emu_tc_trace.argtypes = [vp, dp]
        L.emu_tc_frames.argtypes = [vp, dp]
        L.emu_enable_est.argtypes = [vp, ci]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class TraceSim:
    """one emulated environment on the trace twin's source (traced=False: the chain twin's), with the estimator on and optional frames"""

    def __init__(self, model, fp32=False, frames=None):
        self.L = lib()
        self.h = self.L.emu_tc_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model
        self.L.emu_enable_est(self.h, 1)
        self.nfr = 0
        if frames:
            names, kinds = frames
            arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
            assert self.L.emu_tc_set_frames(self.h, arr, (C.c_int * len(kinds))(*kinds), len(names)) == 0
            self.nfr = len(names)
        self.cols, self.T = [], 0

    def close(self):
        if self.h:
            self.L.emu_tc_free(self.h)
            self.h = None

    def set_trace(self, cols, T):
        src = (C.c_int * max(1, len(cols)))(*[s for s, _ in cols])
        col = (C.c_int * max(1, len(cols)))(*[c for _, c in cols])
        self.L.emu_tc_set_trace(self.h, src, col, len(cols), T)
        self.cols, self.T = list(cols), T

    def traced(self, on):
        self.L.emu_tc_traced(self.h, 1 if on else 0)

    def step(self, row, nticks=1):
        self.L.emu_tc_step(self.h, _dp(np.ascontiguousarray(row, dtype=np.float64)), nticks)

    def forward(self):
        self.L.emu_tc_forward(self.h)

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), _dp(buf), n)
        assert k >= 0, name
        return buf[:k]

    def frames(self):
        buf = np.zeros(64 * FRAME_W)
        return buf[:self.L.emu_tc_frames(self.h, _dp(buf))]

    def trace(self):
        buf = np.zeros(64 * 4096)
        w = self.L.emu_tc_trace(self.h, _dp(buf))
        return buf[:w].reshape(self.T, len(self.cols))

    def rows(self):
        """the traced columns as the rows hold them now (what cassie_batch_get_* returns)"""
        src = {QPOS: self.get('qpos'), QVEL: np.concatenate([self.get('qvel'), self.get('xqvel')]), OBS: self.get('obs'), AUX: self.get('aux'), FRAME: self.frames()}
        return np.array([src[s][c] for s, c in self.cols])


def all_sources(model, nq, nv, nfr, seed=5):
    """64 columns drawn from every source (every column of a short source, both lane passes of the store used)"""
    rng = np.random.default_rng(seed)
    cols = [(QPOS, c) for c in (0, 2, 3, 6, nq - 1)] + [(QVEL, c) for c in (0, 5, 31, nv - 1)]
    cols += [(OBS, c) for c in (0, 20, 29, 42, 55, 56, 60, 86, 96, 99, 105, 111)]
    cols += [(AUX, c) for c in (0, 2, 8, 14, 20, 24, 26, 30, 41, 42, 45, 48, 51, 53, 54)]
    cols += [(FRAME, int(c)) for c in rng.choice(nfr * FRAME_W, 64 - len(cols), replace=False)]
    return cols


def _schedule(k):
    return PD_ROW if k < 4 else ZERO_ROW   # stance, then a fall with the motors off: contacts come and go


# ------------------------------------------------------------------ 1. one 50-tick launch's trace is 50 one-tick launches' rows
@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_trace_equals_one_tick_launches(model, fp32):
    """every source, bitwise, over 8 launches of 50 ticks; the state after each launch equals too, and so does the chain twin's (no trace): the trace
    changes no physics"""
    frames = all_frames(model)
    a, b, c = (TraceSim(model, fp32, frames) for _ in range(3))
    nq, nv = (42, 38) if model == 'cassie_tray_box' else (35, 32)
    cols = all_sources(model, nq, nv, len(frames[0]))
    assert len(cols) == 64
    for s in (a, b, c):
        s.set_trace(cols, 50)
    c.traced(False)
    for k in range(8):
        row = _schedule(k)
        a.step(row, 50)
        c.step(row, 50)
        want = []
        for t in range(50):
            b.step(row, 1)
            want.append(b.rows())
            assert np.array_equal(b.trace()[0], want[-1]), (k, t)   # a one-tick launch writes slot 0
        got = a.trace()
        bad = np.argwhere(got != np.array(want))
        assert bad.size == 0, (k, [(int(t), cols[int(i)]) for t, i in bad[:8]])
        for name in ('qpos', 'qvel', 'xqvel', 'obs', 'aux', 'counters'):
            assert np.array_equal(a.get(name), b.get(name)) and np.array_equal(a.get(name), c.get(name)), (k, name)
        assert np.array_equal(a.frames(), c.frames()), k
    assert a.get('qpos')[2] < 0.95   # the robot is falling
    for s in (a, b, c):
        s.close()


# ------------------------------------------------------------------ 2. against the oracle, every tick
def _state_rows(y):
    """state_out_t fields in the observation row's layout: motor positions (0..9), pelvis acceleration (56..58), pelvis orientation (86..89), the
    estimator's force model and filters (96..111)"""
    return np.concatenate([y.motor.position[:], y.pelvis.translationalAcceleration[:], y.pelvis.orientation[:], y.pelvis.position[:],
                           y.pelvis.translationalVelocity[:], y.pelvis.externalForce[:], [y.terrain.height], y.leftFoot.toeForce[:], y.rightFoot.toeForce[:]])


OBS_COLS = list(range(10)) + [56, 57, 58] + [86, 87, 88, 89] + list(range(96, 112))


def test_trace_follows_the_oracle(oracle_mod, pkg):
    """fp64, 10 launches of 50 ticks, stance then a fall: per tick the foot forces, toe / heel forces, foot positions and velocities within check_row's
    bars (forces 1e-8, positions 1e-10, velocities 1e-8), the centre of mass and the pelvis frame's xquat within 1e-10 of the state the tick started
    from (the rows describe the state the last sub-step started from: test_centre_of_mass_group, test_frames), the state_out_t fields within 1e-10
    relative to 1 + |value| (test_aos_instance's bar) -- two traces of the same run, one of aux and frame columns, one of observation columns.  The
    centre-of-mass velocity and angular momentum need an mj_forward on the oracle's side, which would change its next tick: they are held to the
    one-tick launches bitwise above and to the oracle by test_derived.py"""
    O = oracle_mod
    model = 'cassie'
    o, y = O.OracleSim(os.path.join(GOLDEN, model + '.omodel')), pkg.state_out_t()
    frames = (['cassie-pelvis'], [0])
    a, b = TraceSim(model, False, frames), TraceSim(model, False, frames)
    a.set_trace([(AUX, c) for c in range(45)] + [(FRAME, 3 + i) for i in range(4)], 50)
    b.set_trace([(OBS, c) for c in OBS_COLS] + [(QPOS, c) for c in range(7)], 50)
    stance, off = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    pelvis = 1
    worst = dict(force=0.0, pos=0.0, vel=0.0, cm_pos=0.0, quat=0.0, state=0.0, qpos=0.0)
    for k in range(10):
        row = PD_ROW if k < 5 else ZERO_ROW
        a.step(row, 50)
        b.step(row, 50)
        ta, tb = a.trace(), b.trace()
        for t in range(50):
            cm_pos, quat = o.cm_position(), o.arr('xquat')[4 * pelvis:4 * pelvis + 4].copy()
            o.step_pd(stance if k < 5 else off, y)
            toe, heel = o.heeltoe_forces()
            r = ta[t]
            worst['force'] = max(worst['force'], np.abs(r[0:12] - o.foot_forces()).max(), np.abs(r[12:18] - toe).max(), np.abs(r[18:24] - heel).max())
            worst['pos'] = max(worst['pos'], np.abs(r[24:30] - o.foot_positions()).max())
            worst['vel'] = max(worst['vel'], np.abs(r[30:42] - o.foot_velocities()).max())
            worst['cm_pos'] = max(worst['cm_pos'], np.abs(r[42:45] - cm_pos).max())
            worst['quat'] = max(worst['quat'], np.abs(r[45:49] - quat).max())
            want = _state_rows(y)
            worst['state'] = max(worst['state'], (np.abs(tb[t, :len(OBS_COLS)] - want) / (1 + np.abs(want))).max())
            worst['qpos'] = max(worst['qpos'], np.abs(tb[t, len(OBS_COLS):] - o.arr('qpos')[:7]).max())
    print(worst)
    assert worst['force'] < 1e-8 and worst['pos'] < 1e-10 and worst['vel'] < 1e-8 and worst['cm_pos'] < 1e-10, worst
    assert worst['quat'] < 1e-10 and worst['state'] < 1e-10 and worst['qpos'] < 1e-10, worst
    assert o.arr('qpos')[2] < 0.95   # the robot is falling
    a.close()
    b.close()
    o.close()


# ------------------------------------------------------------------ 3. the slot rules
def test_longer_launches_keep_their_last_ticks():
    """nticks > T keeps the last T ticks in order; nticks < T writes slots 0 .. nticks - 1 and leaves the rest; a forward launch writes nothing"""
    model = 'cassie'
    cols = [(QPOS, 2), (QVEL, 0), (OBS, 20), (AUX, 2)]
    full, short = TraceSim(model), TraceSim(model)
    full.set_trace(cols, 50)
    short.set_trace(cols, 8)
    full.step(PD_ROW, 50)
    short.step(PD_ROW, 50)
    assert np.array_equal(short.trace(), full.trace()[42:])
    before = short.trace()
    full.step(PD_ROW, 5)
    short.step(PD_ROW, 5)
    got = short.trace()
    assert np.array_equal(got[:5], full.trace()[:5]) and np.array_equal(got[5:], before[5:])
    short.forward()
    assert np.array_equal(short.trace(), got)
    full.close()
    short.close()
