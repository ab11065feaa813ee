"""GPU: per-environment placement of the static planes / boxes (cassie_batch_set_env_geom_pose) -- a batch in which every environment has its own
stairs / floor tilt, against one oracle per sampled environment, and the verbs' semantics.  CPU twins (host emulation): tests/test_env_geoms.py."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_env_geoms import placed_oracle
from test_model_variants import STAIRS

pytestmark = pytest.mark.gpu

N = 256


def _layouts(n, seed=7):
    """per environment: kind 0 boxes parked (file placement), 1 a step of height h under each foot, 2 the floor tilted about x and y"""
    rng = np.random.default_rng(seed)
    kind = np.arange(n) % 3
    h = rng.uniform(0.02, 0.06, n)
    yaw = rng.uniform(-0.2, 0.2, n)
    tilt = np.deg2rad(rng.uniform(-3, 3, (n, 2)))
    return kind, h, yaw, tilt


def _placements(kind, h, yaw, tilt):
    """[(name, pos, quat, size)] of one environment (body frame = world frame for these geoms)"""
    if kind == 1:
        q = [np.cos(yaw / 2), 0, 0, np.sin(yaw / 2)]
        return [('box1', [0.05, 0.135, h - 0.1], q, [0.25, 0.1, 0.1]), ('box7', [0.05, -0.135, h - 0.1], q, [0.25, 0.1, 0.1])]
    if kind == 2:
        qx, qy = [np.cos(tilt[0] / 2), np.sin(tilt[0] / 2), 0, 0], [np.cos(tilt[1] / 2), 0, np.sin(tilt[1] / 2), 0]
        q = [qx[0] * qy[0], qx[1] * qy[0], qx[0] * qy[2], qx[1] * qy[2]]
        return [('floor', None, q, None)]
    return []


def _place_batch(b, lay):
    kind, h, yaw, tilt = lay
    for e in range(b.n):
        for name, pos, quat, size in _placements(kind[e], h[e], yaw[e], tilt[e]):
            m = np.zeros(b.n, np.uint8)
            m[e] = 1
            b.set_env_geom_pose(name, pos=pos, quat=quat, size=size, mask=m)


def _oracle(O, placements):
    return placed_oracle(O, placements)


def _pd(P):
    pu = P.pd_in_t()
    for side, leg in enumerate((pu.leftLeg, pu.rightLeg)):
        for i in range(5):
            leg.motorPd.pTarget[i] = PD_TARGET[5 * side + i]
            leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_PGAIN[i], PD_DGAIN[i]
    return pu


@pytest.mark.parametrize('fp64', [True, False])
def test_per_env_layouts_follow_the_oracle(oracle_mod, fp64):
    P, O = product(), oracle_mod
    lay = _layouts(N)
    b = P.CassieBatch(N, precision=P.FP64 if fp64 else P.FP32)
    b.set_pd(P.pd_rows(N, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    _place_batch(b, lay)
    b.forward()
    sample = np.random.default_rng(3).choice(N, 32, replace=False)
    oracles = [_oracle(O, _placements(lay[0][e], lay[1][e], lay[2][e], lay[3][e])) for e in sample]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    iters_ok = True
    for k in range(700):
        b.step(1)
        for o in oracles:
            o.step_pd(u)
        if fp64:
            it = b.counters()[sample, 3]
            iters_ok = iters_ok and all(int(it[i]) == o.get_int('solver_iter') for i, o in enumerate(oracles))
    q = b.qpos()
    err = np.array([np.abs(q[e] - o.arr('qpos')).max() for e, o in zip(sample, oracles)])
    if fp64:
        assert err.max() <= 1e-9 and iters_ok, err.max()
    else:
        assert np.median(err) <= 1e-5 and np.percentile(err, 90) <= 1e-4 and err.max() <= 1e-3, (np.median(err), np.percentile(err, 90), err.max())
    assert int(b.counters()[:, 4].sum()) == 0
    # environments standing on steps stand higher by their step height; the parked / tilted ones stand where a flat-floor environment does
    flat = P.CassieBatch(1, precision=P.FP64)
    flat.set_pd(P.pd_rows(1, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    flat.step(700)
    dz = q[:, 2] - flat.qpos()[0, 2]
    kind, h = lay[0], lay[1]
    print('pelvis height above the flat stance: steps', np.c_[h[kind == 1], dz[kind == 1]][:8], 'parked', np.abs(dz[kind == 0]).max(), 'tilted', np.abs(dz[kind == 2]).max())
    # (the standing controller settles lower on a step: the gain is the step height less a common offset of about 3 cm)
    gain = dz[kind == 1] - h[kind == 1]
    assert np.ptp(gain) < 0.01 and np.corrcoef(h[kind == 1], dz[kind == 1])[0, 1] > 0.95 and (dz[kind == 1][h[kind == 1] > 0.045] > 0.01).all(), np.c_[h[kind == 1], dz[kind == 1]]
    assert np.abs(dz[kind == 0]).max() < 1e-6 and np.abs(dz[kind == 2]).max() < 0.01


def test_equal_rows_equal_the_shared_placement():
    P = product()
    n = 64
    a, b = P.CassieBatch(n, precision=P.FP64), P.CassieBatch(n, precision=P.FP64)
    rows = P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    a.set_pd(rows)
    b.set_pd(rows)
    for name, pos, quat, size in STAIRS:
        a.set_geom_pose(name, pos=pos, quat=quat, size=size)
        b.set_env_geom_pose(name, pos=pos, quat=quat, size=size)
    a.forward()
    b.forward()
    for k in range(600):
        a.step(1)
        b.step(1)
        ca, cb = a.counters(), b.counters()
        assert np.array_equal(ca[:, :5], cb[:, :5]), k   # constraint rows, contacts, limits, iterations, drops
    assert np.abs(a.qpos() - b.qpos()).max() <= 1e-9


@pytest.mark.parametrize('fp64', [True, False])
def test_aos_entry_point_matches_the_compact_path(fp64):
    """cassie_sim_step_pd_batch runs the plain + estimator instance (f2c / d2f), the compact path the plain one (f0c / d0f)"""
    P = product()
    n = 96
    lay = _layouts(n, seed=11)
    a, b = (P.CassieBatch(n, precision=P.FP64 if fp64 else P.FP32) for _ in range(2))
    _place_batch(a, lay)
    _place_batch(b, lay)
    a.forward()
    b.forward()
    pu = (P.pd_in_t * n)(*([_pd(P)] * n))
    a.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    for k in range(300):
        a.step(1)
        b.step_pd(pu, want_state=False)
    assert np.abs(a.qpos() - b.qpos()).max() <= (1e-9 if fp64 else 1e-4)
    assert np.array_equal(a.counters()[:, 4], b.counters()[:, 4])


def test_derived_quantities_follow_each_environment(oracle_mod):
    P, O = product(), oracle_mod
    n = 12
    lay = _layouts(n, seed=5)
    b = P.CassieBatch(n, precision=P.FP64)
    b.enable_aux()
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    _place_batch(b, lay)
    b.forward()
    oracles = [_oracle(O, _placements(lay[0][e], lay[1][e], lay[2][e], lay[3][e])) for e in range(n)]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for k in range(400):
        b.step(1)
        for o in oracles:
            o.step_pd(u)
    aux = b.aux()
    for e, o in enumerate(oracles):
        assert np.abs(aux[e, 0:12] - o.foot_forces()).max() < 1e-6, e
        mask = sum(1 << g for g in range(16) if o.geom_collision(g))
        assert int(aux[e, 53]) == mask, (e, int(aux[e, 53]), mask)


def test_verb_semantics():
    P = product()
    n = 8
    b = P.CassieBatch(n, precision=P.FP32)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    pos0, quat0, size0 = b.env_geom_pose('box1')   # no rows yet: the shared placement
    assert (pos0 == pos0[0]).all() and np.allclose(size0, 1.0)
    # a masked set changes only the selected environments
    m = np.array([1, 0, 1, 0, 0, 0, 0, 0], np.uint8)
    b.set_env_geom_pose('box1', pos=[0.05, 0.135, -0.05], size=[0.25, 0.1, 0.1], mask=m)
    pos, quat, size = b.env_geom_pose('box1')
    assert np.allclose(pos[m == 1], [0.05, 0.135, -0.05]) and np.array_equal(pos[m == 0], pos0[m == 0]) and np.array_equal(quat, quat0)
    assert np.allclose(size[m == 1], [0.25, 0.1, 0.1]) and np.array_equal(size[m == 0], size0[m == 0])
    b.set_env_geom_pose('box1', quat=[np.cos(0.1), 0, 0, np.sin(0.1)], mask=m)   # a None part is left alone
    pos2, quat2, _ = b.env_geom_pose('box1')
    assert np.array_equal(pos2, pos) and np.allclose(quat2[m == 1], [np.cos(0.1), 0, 0, np.sin(0.1)])
    b.step(300)
    z = b.qpos()[:, 2]
    assert (z[m == 1] - z[m == 0].max() > 0.005).all() and np.ptp(z[m == 0]) < 1e-6   # a 5 cm step under the left foot lifts the selected environments only
    # reset and snapshot restore leave the placement alone
    snap = b.get_state()
    b.reset()
    assert np.array_equal(b.env_geom_pose('box1')[0], pos2)
    b.step(300)
    assert np.abs(b.qpos()[:, 2] - z).max() < 1e-6
    b.set_state(snap)
    assert np.array_equal(b.env_geom_pose('box1')[0], pos2)
    b.free_state(snap)
    # the shared verb after rows exist rewrites that geom's slot in every environment
    b.set_geom_pose('box1', pos=[0.05, 0.135, -0.08], size=[0.25, 0.1, 0.1])
    pos3, _, _ = b.env_geom_pose('box1')
    assert np.allclose(pos3, [0.05, 0.135, -0.08]) and np.allclose(b.env_geom_pose('box1')[1], [1, 0, 0, 0])
    b.reset()
    b.step(300)
    z3 = b.qpos()[:, 2]
    assert np.ptp(z3) < 1e-5
    # the error cases return -1 and change nothing
    L = P.lib()
    one = np.zeros((n, 3))
    assert L.cassie_batch_set_env_geom_pose(b.h, b'no-such-geom', b._dp(one), None, None, None) == -1   # (the robot's geoms carry no names in cassie.xml)
    assert np.array_equal(b.env_geom_pose('box1')[0], pos3)
    with pytest.raises(RuntimeError):
        b.env_geom_pose('no-such-geom')
    # clear: the shared placement again (box1 at -0.08 under the left foot for every environment, as the shared verb set it)
    pos7 = b.env_geom_pose('box7')[0]
    b.set_env_geom_pose('box7', pos=[0.05, -0.135, -0.05], size=[0.25, 0.1, 0.1], mask=m)
    b.clear_env_geom_poses()
    assert np.array_equal(b.env_geom_pose('box7')[0], pos7)
    b.reset()
    b.step(300)
    assert np.abs(b.qpos()[:, 2] - z3).max() < 1e-6
    b.close()


def test_height_field_is_refused():
    P = product()
    b = P.CassieBatch(4, modelfile=P.model_path('cassie_hfield'), precision=P.FP32)
    assert P.lib().cassie_batch_set_env_geom_pose(b.h, b'hfield1', None, None, None, None) == -1 and 'height field' in P._last_error()
    with pytest.raises(RuntimeError):
        b.env_geom_pose('hfield1')
    b.close()
