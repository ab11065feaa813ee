"""The mass-matrix factorisation generated for the Cassie dof tree (tools/gen_tree_code.py -> CT19_FACTOR) against the table-driven one it replaces on
that tree: both factor_ld paths of the product source run on the host (tests/emu/emu_factor.cpp, -DCASSIE_EMU) on the same M and M + hB, taken from the
emulated stepper's debug dump at a standing, a fallen and a tray-carrying state.  They apply the same multiply-subtracts in the same order, so every
entry of both factors, 1/D, 1/sqrt(D) and the second matrix's 1/D must be bitwise equal, in both precisions."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET

import emu_harness as E

PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
_lib = None


def lib():
    global _lib
    if _lib is None:
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_factor.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_factor.cpp'), os.path.join(E.CSRC, 'mjcf.cpp')] + [os.path.join(E.CSRC, f) for f in (
            'step_core.inl', 'cassie_tree_gen.inc', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h')]
        if not os.path.exists(out) or any(os.path.getmtime(s) > os.path.getmtime(out) for s in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], srcs[1]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        dp = C.POINTER(C.c_double)
        L.emu_factor.argtypes = [C.c_char_p, C.c_int, C.c_int, dp, dp, dp, dp, dp, dp, dp]
        _lib = L
    return _lib


def dof_madr(model):
    """the main tree's dof_Madr (the diagonal entries of M) from the compiled model table"""
    for line in open(model):
        if line.startswith('dof_Madr I '):
            f = line.split()
            return np.array([int(x) for x in f[3:3 + int(f[2])]])[:32]
    raise AssertionError('no dof_Madr in ' + model)


def mass_matrix(model, pd, ticks):
    """M at the state reached after `ticks` ticks of the emulated stepper under the PD row `pd` (fp64), from its debug dump"""
    s = E.EmuSim(model)
    s.step(pd, ticks)
    m = s.get('dbg')[E.D['QM']:E.D['QLD']].copy()
    s.close()
    return m


def factor(model, fp32, spec, m, m2):
    n = m.size
    out, out2, dinv, dsqi, dinv2 = np.zeros(n), np.zeros(n), np.zeros(32), np.zeros(32), np.zeros(32)
    p = lambda a: a.ctypes.data_as(C.POINTER(C.c_double))
    nm = lib().emu_factor(model.encode(), 1 if fp32 else 0, spec, p(m), None if m2 is None else p(m2), p(out), p(out2), p(dinv), p(dsqi), p(dinv2))
    assert nm > 0, nm
    return out[:nm], out2[:nm], dinv, dsqi, dinv2


STATES = {'stance': ('cassie', PD_ROW, 300), 'fall': ('cassie', np.zeros(50), 600), 'tray_box': ('cassie_tray_box', PD_ROW, 300)}


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('state', sorted(STATES))
def test_generated_factor_is_bitwise_the_table_factor(pkg, state, fp32):
    name, pd, ticks = STATES[state]
    model = pkg.model_path(name)
    m = mass_matrix(model, pd, ticks)
    assert np.isfinite(m).all() and np.abs(m).max() > 0
    # the second matrix is M with a heavier diagonal, as M + h B is
    m2 = m.copy()
    m2[dof_madr(model)] += 5e-4 * (1 + np.arange(32) % 3)
    want = factor(model, fp32, 0, m, m2)
    got = factor(model, fp32, 1, m, m2)
    for w, g, what in zip(want, got, ('L of M', 'L of M + hB', '1/D', '1/sqrt(D)', '1/D of M + hB')):
        assert np.array_equal(w.view(np.uint64), g.view(np.uint64)), (state, what, np.flatnonzero(w != g)[:8])
    # M alone (a step without damping): the upper lanes idle and the first factor is unchanged
    alone_w, alone_g = factor(model, fp32, 0, m, None), factor(model, fp32, 1, m, None)
    for w, g in zip(alone_w[0:1] + alone_w[2:4], alone_g[0:1] + alone_g[2:4]):
        assert np.array_equal(w.view(np.uint64), g.view(np.uint64)), state
    assert np.array_equal(alone_g[0].view(np.uint64), got[0].view(np.uint64))
