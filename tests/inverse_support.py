"""Inverse dynamics (mj_inverse of MuJoCo 2.1.0, continuous time) restated on the fp64 oracle, for tests/test_inverse.py and tests/test_gpu_inverse.py.

The oracle is forward()ed at the state; everything the inverse needs at that state is then in its arrays, none of which depends on qacc: the sparse qM
(expanded with mj_fullM), qfrc_bias, qfrc_passive and the constraint rows efc_J, efc_aref and efc_D = 1 / efc_R, in MuJoCo's order (the 3 neq rows of
the connect equalities first, then limits and contacts, all inequalities).  At the caller's qacc:
    jar = J qacc - aref;  f = -D jar, and f = 0 on an inequality row with jar >= 0;  qfrc_constraint = J' f;
    qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint.
The oracle runs with the product's capacities (12 contacts, 48 rows), so that both see the same rows."""
import ctypes as C
import os

import numpy as np

from conftest import GOLDEN
from mechanics_support import oracle_with
from test_dynamics import full_m
from test_frames import omodel

COLS, QFRC, QFRCC, NEFC, NCON, DROPPED, WIDTH = 40, 0, 40, 80, 81, 82, 96


def oracle_at(O, model, qpos, qvel, hfield=None, **lines):
    """an fp64 oracle of `model` at (qpos, qvel), forward()ed with zero ctrl and no applied forces; lines: model-table arrays by name (as
    mechanics_support.oracle_with takes them), hfield: the height field's elevations"""
    o = oracle_with(O, model, **lines) if lines else O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    if hfield is not None:
        C.memmove(o.L.osim_hfield_data(o.h), hfield.ctypes.data, hfield.nbytes)
    o.set_caps(12, 48)
    o.arr('qpos')[:] = qpos[:o.nq]
    o.arr('qvel')[:] = qvel[:o.nv]
    o.forward()
    return o


def inverse(o, model, qacc):
    """the restatement at the oracle's current (forward()ed) state and qacc [nv]: qfrc_inverse, qfrc_constraint, the row forces f and their jar, the
    inequality flags, nefc and ncon"""
    m = omodel(model)
    nv, neq, nefc = o.nv, m['eq_obj1id'].size, o.get_int('nefc')
    qacc = np.asarray(qacc, float)[:nv]
    M = full_m(o.arr('qM'), m)
    J = o.efc_J()
    jar = J @ qacc - o.arr('efc_aref')
    f = -o.arr('efc_D') * jar
    ineq = np.arange(nefc) >= 3 * neq
    f[ineq & (jar >= 0)] = 0
    qc = J.T @ f
    Mq, bp = M @ qacc, o.arr('qfrc_bias') - o.arr('qfrc_passive')
    inv = Mq + bp - qc
    return dict(qfrc_inverse=inv, qfrc_constraint=qc, f=f, jar=jar, ineq=ineq, nefc=nefc, ncon=o.get_int('ncon'),
                terms=max(np.abs(Mq).max(), np.abs(bp).max(), np.abs(qc).max()))


def scale(want):
    """the size an error is measured against: the largest entry of the three terms qfrc_inverse is the sum of (M qacc, qfrc_bias - qfrc_passive,
    qfrc_constraint).  qfrc_inverse itself can be near zero while they are not: at a solved qacc without torques it is what the forward applied"""
    return max(1e-300, want['terms'])


def unpack(row, nv):
    """an inverse row [WIDTH] (the emulation's or the batch's device row) in the shapes of cassie_batch_get_inverse"""
    return dict(qfrc_inverse=row[QFRC:QFRC + nv], qfrc_constraint=row[QFRCC:QFRCC + nv], nefc=int(row[NEFC]), ncon=int(row[NCON]), dropped=int(row[DROPPED]))


def columns(qacc, nv):
    """qacc [nv] as a row of the batch's "inv_qacc" layout [COLS] (main tree 0..31, the extra free body 32..37)"""
    out = np.zeros(COLS)
    out[:nv] = qacc[:nv]
    return out
