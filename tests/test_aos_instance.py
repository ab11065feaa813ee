"""The kernel instance cassie_sim_step_pd_batch runs (plain instance + estimator stage, INST 2 in step_kernel.cuh), executed on the host
(tests/emu/emu_aos.cpp, -DCASSIE_EMU): bitwise equal to the extended instance with its estimator, and equal to the oracle's twin estimator to rounding.

Trajectory: 600 ticks of the standing controller, a pelvis push for 60 ticks, then the motors off and a fall; launches of 1 and of 4 ticks.
The plain instance has no extended tail in its scratch: the emulation fills that tail with NaN, so a stage that reads it shows up here."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET

OMODEL = os.path.join(GOLDEN, 'cassie.omodel')
STANCE_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
PUSH = np.array([120.0, -70.0, 40.0, 0, 0, 0])
STAND, PUSHED, TICKS = 600, 660, 900      # stance until STAND, pelvis push until PUSHED, motors off until TICKS


def _launches(e, nt):
    """step emulation e through the schedule in launches of nt ticks; yields the tick count after each launch"""
    for k in range(0, TICKS, nt):
        if k == STAND:
            e.set('xfrc', np.concatenate([PUSH, [1, 0]]))
        if k == PUSHED:
            e.set('xfrc', np.zeros(8))
        e.step(STANCE_ROW if k < PUSHED else np.zeros(50), nt)
        yield k + nt


class AosEmu:
    """the plain instance with the estimator stage: emu.cpp's handle, stepped through emu_aos.cpp"""

    def __init__(self, model_path, fp32):
        import emu_harness as E
        lib = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_aos.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_aos.cpp'), os.path.join(E.HERE, 'emu', 'emu.cpp'), os.path.join(E.CSRC, 'mjcf.cpp'),
                os.path.join(E.CSRC, 'step_core.inl'), os.path.join(E.CSRC, 'devmodel.h'), os.path.join(E.CSRC, 'devbuild.h'), os.path.join(E.CSRC, 'model.h'),
                os.path.join(E.CSRC, 'estimator_host.h'), os.path.join(E.CSRC, 'cassie_tree_gen.inc')]
        if not os.path.exists(lib) or any(os.path.getmtime(lib) < os.path.getmtime(s) for s in srcs):
            os.makedirs(os.path.dirname(lib), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', lib + '.tmp', srcs[0], srcs[2]])
            os.replace(lib + '.tmp', lib)
        self.L = L = C.CDLL(lib)
        dp = C.POINTER(C.c_double)
        L.emu_new.restype = C.c_void_p
        L.emu_new.argtypes = [C.c_char_p, C.c_int]
        L.emu_free.argtypes = [C.c_void_p]
        L.emu_aos_start.argtypes = [C.c_void_p]
        L.emu_aos_step.argtypes = [C.c_void_p, dp, C.c_int]
        L.emu_get.argtypes = L.emu_set.argtypes = [C.c_void_p, C.c_char_p, dp, C.c_int]
        self.h = L.emu_new(model_path.encode(), 1 if fp32 else 0)
        assert self.h, model_path
        L.emu_aos_start(self.h)

    def step(self, pd50, nticks=1):
        a = np.ascontiguousarray(pd50, dtype=np.float64)
        self.L.emu_aos_step(self.h, a.ctypes.data_as(C.POINTER(C.c_double)), nticks)

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def set(self, name, arr):
        a = np.ascontiguousarray(arr, dtype=np.float64)
        assert self.L.emu_set(self.h, name.encode(), a.ctypes.data_as(C.POINTER(C.c_double)), a.size) >= 0

    def close(self):
        if self.h:
            self.L.emu_free(self.h)
            self.h = None


def _emu(pkg, fp32, plain):
    if plain:
        return AosEmu(pkg.model_path('cassie'), fp32)
    from emu_harness import EmuSim
    e = EmuSim(pkg.model_path('cassie'), fp32=fp32)
    e.enable_est()
    return e


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('nt', [1, 4])
def test_plain_estimator_instance_equals_extended_bitwise(pkg, fp32, nt):
    """qpos, qvel and the whole observation row (estimator columns included) after every launch"""
    a, b = _emu(pkg, fp32, True), _emu(pkg, fp32, False)
    for k, _ in zip(_launches(a, nt), _launches(b, nt)):
        for name in ('qpos', 'qvel', 'obs'):
            assert np.array_equal(a.get(name), b.get(name)), (name, k)
    eo, q = a.get('est_out'), a.get('qpos')
    assert np.isfinite(eo).all() and np.abs(eo).max() > 1 and q[2] < 0.8, (eo, q[2])     # the estimator ran; the robot fell
    a.close(); b.close()


@pytest.mark.parametrize('nt', [1, 4])
def test_plain_estimator_instance_matches_oracle(oracle_mod, pkg, nt):
    """fp64, against the oracle's restated estimator: qpos within 1e-10, the estimator outputs within 1e-10 relative to 1 + |a| -- the bars of
    test_emu_parity.py::test_in_kernel_estimator_matches_oracle"""
    O = oracle_mod
    o, y, e = O.OracleSim(OMODEL), pkg.state_out_t(), _emu(pkg, False, True)
    stance, off = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()

    def rows(y):
        return np.concatenate([y.pelvis.position[:], y.pelvis.translationalVelocity[:], y.pelvis.externalForce[:], [y.terrain.height],
                               y.leftFoot.toeForce[:], y.rightFoot.toeForce[:]])
    t, wq, we, fz = 0, 0.0, 0.0, 0.0
    for k in _launches(e, nt):
        for _ in range(k - t):
            if t == STAND:
                o.arr('xfrc_applied').reshape(-1, 6)[1] = PUSH
            if t == PUSHED:
                o.arr('xfrc_applied')[:] = 0
            o.step_pd(stance if t < PUSHED else off, y)
            t += 1
        a = rows(y)
        wq = max(wq, float(np.abs(e.get('qpos')[:35] - o.arr('qpos')).max()))
        we = max(we, float((np.abs(a - e.get('est_out')) / (1 + np.abs(a))).max()))
        fz = max(fz, abs(float(a[6])))
    assert wq < 1e-10 and we < 1e-10, (nt, wq, we)
    assert fz > 10 and o.arr('qpos')[2] < 0.8, (fz, o.arr('qpos')[2])     # the push moved the estimated external force; the robot fell
    e.close()
