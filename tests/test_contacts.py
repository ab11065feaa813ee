"""Contact lists (cassie_batch_enable_contacts): the product's stepper source in the host emulation with a contact-list row, i.e. the F_CL instances,
against the numpy restatement over the fp64 oracle (tests/contact_list_support.py), the aux and frame rows of the same sub-step, and the chain twin it is
the twin of.  The GPU twins are in tests/test_gpu_contacts.py.

Each comparison places a fresh oracle and the emulated environment at one oracle state (qpos, qvel, warm start) and runs one forward on each, so that
both list the contacts of the same state."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET
from contact_list_support import (CON_HEAD, CON_SLOT, DIM, EFC, FORCE, GEOM1, GEOM2, ListSim, compare, restate, slots, table, world_forces)

PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
ZERO_ROW = np.zeros(50)
# fp32 bars, set from the measured distribution over the states below (largest seen: geometry 1.1e-6 of its scale, forces 4.1e-4 of the largest
# force, cassie_tray_box), as DESIGN.md section 3 "Tolerances" sets the other fp32 bars
FP32_GEO, FP32_FORCE = 1e-5, 3e-3


def _states(O, model, ticks=2400, every=160):
    """(qpos, qvel, qacc_warmstart) of the oracle through stance, a gait (targets swinging the hips) and a fall"""
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    out = []
    for k in range(ticks):
        if k < ticks // 3:
            u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
        elif k < 2 * ticks // 3:
            t = np.array(PD_TARGET, float)
            s = 0.3 * np.sin(2 * np.pi * 1.5 * k * 5e-4)
            t[2] += s
            t[7] -= s
            u = O.make_pd(pTarget=list(t), pGain=PD_PGAIN, dGain=PD_DGAIN)
        else:
            u = O.make_pd()
        o.step_pd(u)
        if k % every == every - 1:
            out.append((o.arr('qpos').copy(), o.arr('qvel').copy(), o.arr('qacc_warmstart').copy()))
    o.close()
    return out


def _placed(O, model, state, fp32, friction=None, path=None, setup=None, caps=None):
    """(emulated row, restated row, emulated simulator) after one forward of each at `state`"""
    q, v, ws = state
    t = table(model)
    o = O.OracleSim(path or os.path.join(GOLDEN, model + '.omodel'))
    if caps:
        o.set_caps(*caps)
    if friction is not None:
        o.model_arr('geom_friction')[0::3] = friction
    o.arr('qpos')[:] = q
    o.arr('qvel')[:] = v
    o.arr('qacc_warmstart')[:] = ws
    d0 = o.get_int('dropped_contacts')
    o.forward()
    found = len(o.contacts()) + o.get_int('dropped_contacts') - d0
    want = restate(o, t, friction, found)
    o.close()
    e = ListSim(model, fp32)
    if friction is not None:
        e.model_set('geom_friction', np.repeat(friction, 3))
    if setup:
        setup(e)
    e.place(q, v, ws)
    e.forward()
    return e.row(), want, e


def _check(got, want, fp32, geo_bar=1e-12):
    exact, geo, force = compare(got, want)
    assert exact, (got[:3], want[:3], slots(got)[:, [GEOM1, GEOM2, DIM]].tolist(), slots(want)[:, [GEOM1, GEOM2, DIM]].tolist())
    if fp32:
        assert geo < FP32_GEO and force < FP32_FORCE, (geo, force)
    else:
        assert geo < geo_bar and force < 1e-8, (geo, force)
    return geo, force


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box', 'cassie_depth'])
def test_contacts_follow_the_oracle(oracle_mod, model, fp32):
    """stance, gait and fall states: geom ids, condim, efc addresses and counts exact; positions, frames and depths within 1e-12 of their scale and
    forces within 1e-8 of the largest force (fp64), the fp32 bars above"""
    worst, listed = [0.0, 0.0], 0
    for state in _states(oracle_mod, model):
        got, want, e = _placed(oracle_mod, model, state, fp32)
        e.close()
        g, f = _check(got, want, fp32)
        worst = [max(worst[0], g), max(worst[1], f)]
        listed = max(listed, int(want[0]))
    print(model, 'fp32' if fp32 else 'fp64', 'geometry %.3g force %.3g' % tuple(worst), 'most listed', listed)
    assert listed >= 2


def test_box_and_floor_contacts_in_mujoco_order(oracle_mod):
    """a stair box moved under one foot: the list holds box and floor contacts of both collision runs in MuJoCo's order, as the oracle lists them"""
    from test_env_geoms import STAIRS, placed_oracle
    O = oracle_mod
    name, pos, _, size = STAIRS[0]
    o = placed_oracle(O, [(name, pos, None, size)])
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    mixed = 0
    for k in range(400):
        o.step_pd(u)
        gs = [c['geom1'] for c in o.contacts()]
        if k % 20 == 19 and 0 in gs and any(x != 0 for x in gs) and gs != sorted(gs):
            state = (o.arr('qpos').copy(), o.arr('qvel').copy(), o.arr('qacc_warmstart').copy())
            for fp32 in (False, True):
                q, v, ws = state
                p = placed_oracle(O, [(name, pos, None, size)])
                p.arr('qpos')[:] = q
                p.arr('qvel')[:] = v
                p.arr('qacc_warmstart')[:] = ws
                p.forward()
                want = restate(p, table('cassie'))
                p.close()
                e = ListSim('cassie', fp32)
                e.set_geom(name, pos=pos, size=size)
                e.place(q, v, ws)
                e.forward()
                _check(e.row(), want, fp32)
                e.close()
            mixed += 1
    o.close()
    assert mixed >= 3, mixed


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_per_environment_friction(oracle_mod, model):
    """per-environment friction rows: the slots' mu and the decoded tangential forces follow the oracle with the same geom friction"""
    t = table(model)
    friction = np.array(t['geom_friction'], float)[0::3].copy()
    friction[:] = np.where(friction > 0, 0.35, friction)
    friction[0] = 0.6   # the floor
    n = 0
    for state in _states(oracle_mod, model, ticks=300, every=100):
        got, want, e = _placed(oracle_mod, model, state, False, friction=friction)
        e.close()
        _check(got, want, False)
        n += int(want[0])
    assert n > 0


def test_capacity_drops_like_the_oracle(oracle_mod):
    """lying face down on the floor with every resting body touching (11 contacts): listed, found and dropped as the oracle with the product's
    capacities (set_caps(12, 48)) counts them, and the listed slots as it lists them -- the 48 rows hold the 12 equality rows and 9 pyramidal contacts"""
    O = oracle_mod
    o = O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    q, v, ws = o.arr('qpos').copy(), o.arr('qvel').copy(), o.arr('qacc_warmstart').copy()
    o.close()
    q[2], q[3:7] = 0.0, [np.cos(np.pi / 4), 0, np.sin(np.pi / 4), 0]
    got, want, e = _placed(O, 'cassie', (q, v, ws), False, caps=(12, 48))
    e.close()
    _check(got, want, False, geo_bar=1e-11)   # bodies sunk into the floor by centimetres: the capsule-plane geometry rounds a few ulps apart
    assert list(want[:3]) == [9, 11, 2] and slots(want)[8, EFC] == 44, want[:3]


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_listed_forces_sum_to_the_aux_and_frame_rows(model, fp32):
    """the signed foot sums of the listed world forces are the aux row's foot forces, their toe / heel split its toe and heel forces' total, and
    the body sums the frame rows' CFRC, after 50-tick launches through stance and a fall"""
    from test_frames import all_frames
    names, kinds = all_frames(model)
    e = ListSim(model, fp32, (names, kinds))
    t = table(model)
    body = [int(x) for x in t['geom_bodyid']]
    lf, rf = t['names_body'].index('left-foot'), t['names_body'].index('right-foot')
    tol = 1e-5 if fp32 else 1e-12
    seen = 0
    for k in range(8):
        e.step(PD_ROW if k < 4 else ZERO_ROW, 50)
        row, aux, fr = e.row(), e.get('aux'), e.frames().reshape(-1, 20)
        s, w = slots(row)[:int(row[0])], world_forces(row)
        feet = np.zeros(12)
        tot = np.zeros(len(names) * 3).reshape(-1, 3)
        for c in range(len(s)):
            b1, b2 = body[int(s[c, GEOM1])], body[int(s[c, GEOM2])]
            for side, fb in enumerate((lf, rf)):
                feet[6 * side:6 * side + 3] += (w[c] if b2 == fb else 0) - (w[c] if b1 == fb else 0)
            for f, (nm, kd) in enumerate(zip(names, kinds)):
                if kd == 0:
                    bi = t['names_body'].index(nm)
                    tot[f] += (w[c] if b2 == bi else 0) - (w[c] if b1 == bi else 0)
        scale = max(1.0, np.abs(aux[0:12]).max())
        assert np.abs(feet - aux[0:12]).max() < tol * scale, (k, feet, aux[0:12])
        toeheel = aux[12:18] + aux[18:24]
        assert np.abs(toeheel - feet[[0, 1, 2, 6, 7, 8]]).max() < tol * scale, k
        assert np.abs(tot - fr[:, 13:16]).max() < tol * max(1.0, np.abs(fr[:, 13:16]).max()), k
        seen += len(s)
    e.close()
    assert seen > 8


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_lists_change_no_physics(model, fp32):
    """the F_CL source and the chain twin's, stepped alike with a per-environment body offset in the rows: state, observation, aux, counters and frame
    rows bitwise equal after every single-tick and 50-tick launch; query and dynamics launches leave the list alone, a forward launch refills it"""
    from test_frames import all_frames
    frames = all_frames(model)
    a, b = ListSim(model, fp32, frames), ListSim(model, fp32, frames)
    b.listed(False)
    t = table(model)
    bp = np.array(t['body_pos'], float)
    bp[3 * t['names_body'].index('left-foot'):][:3] *= 1.01
    for s in (a, b):
        s.rows_set('bp', bp)
    for k in range(6):
        for nticks in (1, 50):
            a.step(PD_ROW if k < 3 else ZERO_ROW, nticks)
            b.step(PD_ROW if k < 3 else ZERO_ROW, nticks)
            for name in ('qpos', 'qvel', 'xqvel', 'qacc_ws', 'obs', 'aux', 'counters', 'cst'):
                assert np.array_equal(a.get(name), b.get(name)), (k, nticks, name)
            assert np.array_equal(a.frames(), b.frames()), (k, nticks)
    row = a.row()
    assert row[0] > 0
    for mode in (2, 5):   # query, dynamics
        a.mode(mode)
        assert np.array_equal(a.row(), row), mode
    a.forward()
    assert a.row()[1] >= a.row()[0] > 0
    a.close()
    b.close()
