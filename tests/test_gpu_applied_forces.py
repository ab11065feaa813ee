"""GPU: per-environment applied forces (cassie_batch_set_applied_forces, the F_XF instances: xfrc_applied per body, qfrc_applied per dof), against the
fp64 oracle given the same arrays, and the verbs' behaviour: masks, validation, reset, clear_forces, snapshots, the legacy simulator and the device rows."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO, product
from mechanics_support import oracle_with, random_mechanics, table
from test_applied_forces import schedule
from test_gpu_configs import BARS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def P():
    return product()


def _pd(P, b, n):
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))


def _oracle(O, model, **lines):
    o = oracle_with(O, model, **lines) if lines else O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    o.set_caps()
    return o


def test_four_envs_fp64(P, oracle_mod):
    """4 environments with their own rows, one also with mechanics rows and one with a floor tilt (d17df), against 4 oracles: qpos within 1e-9 and equal
    PGS iteration counts over 500 ticks"""
    O, n, model = oracle_mod, 4, 'cassie'
    t = table(model)
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    nb, nv = b.L.cassie_batch_nbody(b.h), b.nv
    scheds = [schedule(model, 70 + e, nb, nv) for e in range(n)]
    inertia, armature, stiffness, springref = random_mechanics(model, 5)
    b.set_env_mechanics(inertia, armature, stiffness, springref, mask=np.array([0, 1, 0, 0], np.uint8))
    tilt = np.array([np.cos(0.01), np.sin(0.01), 0.0, 0.0])
    b.set_env_geom_pose('floor', quat=np.array([[1.0, 0, 0, 0], [1.0, 0, 0, 0], tilt, [1.0, 0, 0, 0]]))
    gq = t['geom_quat'].reshape(-1, 4).copy()
    gq[0] = tilt
    os_ = [_oracle(O, model), oracle_with(O, model, inertia=inertia, armature=armature, stiffness=stiffness, springref=springref), _oracle(O, model, geom_quat=gq), _oracle(O, model)]
    os_[1].set_caps()
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    _pd(P, b, n)
    b.reset()
    for o in os_:
        o.forward()
    same, worst = True, 0.0
    for k in range(5):
        b.set_applied_forces(np.stack([s[k][0] for s in scheds]), np.stack([s[k][1] for s in scheds]))
        for e, o in enumerate(os_):
            o.arr('xfrc_applied')[:] = scheds[e][k][0].ravel()
            o.arr('qfrc_applied')[:] = scheds[e][k][1]
        for _ in range(100):
            b.step(1)
            it, q = b.counters()[:, 3], b.qpos()
            for e, o in enumerate(os_):
                o.step_pd(u)
                same = same and int(it[e]) == o.get_int('solver_iter')
                worst = max(worst, float(np.abs(q[e, :o.nq] - o.arr('qpos')).max()))
    print('four fp64 environments with applied forces: worst qpos %.2e' % worst)
    assert worst < 1e-9 and same, (worst, same)
    for o in os_:
        o.close()
    b.close()


def test_tray_box_cup_pushes_fp64(P, oracle_mod):
    """cassie_tray_box: pushes on the cup (the extra free body) and qfrc on its dofs, with the rest of the schedule, against the oracle over 500 ticks"""
    O, model = oracle_mod, 'cassie_tray_box'
    b = P.CassieBatch(2, modelfile=P.model_path(model), precision=P.FP64)
    nb, nv = b.L.cassie_batch_nbody(b.h), b.nv
    sched = schedule(model, 17, nb, nv)
    o = _oracle(O, model)
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    _pd(P, b, 2)
    b.reset()
    o.forward()
    same, worst = True, 0.0
    for x, q in sched:
        b.set_applied_forces(x, q)
        o.arr('xfrc_applied')[:] = x.ravel()
        o.arr('qfrc_applied')[:] = q
        for _ in range(100):
            b.step(1)
            o.step_pd(u)
            same = same and int(b.counters()[0, 3]) == o.get_int('solver_iter')
            worst = max(worst, float(np.abs(b.qpos()[0, :o.nq] - o.arr('qpos')).max()))
    print('tray box with cup pushes: worst qpos %.2e' % worst)
    assert worst < 1e-9 and same, (worst, same)
    o.close()
    b.close()


def test_fp32_4096_push_schedule_through_the_device_rows(P, oracle_mod):
    """4096 fp32 cassie.xml environments on the plain twin (f0404): config 3's Philox pushes written through torch_view('applied'), alternating the pelvis
    (even events) and the left foot (odd events), held 100 ticks of every 400; 64 sampled environments replayed in the oracle within config 3's bars"""
    import torch
    sys.path.insert(0, REPO)
    import bench
    old = os.environ.pop('CASSIE_B200_DEBUG', None)
    try:
        O, n, T, model = oracle_mod, 4096, 600, 'cassie'
        b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32)
        names = table(model)['names_body']
        body = [names.index('cassie-pelvis'), names.index('left-foot')]
        b.enable_applied_forces()
        _pd(P, b, n)
        b.reset()
        b.set_stream(torch.cuda.current_stream().cuda_stream)
        view = b.torch_view('applied')
        q_init = b.qpos()
        sample = np.sort(np.random.default_rng(7).choice(n, 64, replace=False))
        got = []
        for t in range(T):
            if t % 400 == 0:
                k = t // 400
                push = torch.as_tensor(bench.philox_uniform(1234, k, (n, 2), -100.0, 100.0) * (1.0 if k % 2 == 0 else 0.2), dtype=torch.float32, device='cuda')
                view[:, 6 * body[k % 2]:6 * body[k % 2] + 2] = push
            elif t % 400 == 100:
                view[:, :192] = 0
            b.step(1)
            if (t + 1) % 100 == 0:
                got.append(b.qpos()[sample])
        assert b.launch_count() > 0
        got = np.array(got)
        err = np.zeros(len(sample))
        for j, e in enumerate(sample):
            o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
            o.arr('qpos')[:o.nq] = q_init[e]
            o.forward()
            u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
            want = []
            for t in range(T):
                if t % 400 == 0:
                    k = t // 400
                    o.arr('xfrc_applied').reshape(-1, 6)[body[k % 2], :2] = bench.philox_uniform(1234, k, (n, 2), -100.0, 100.0)[e] * (1.0 if k % 2 == 0 else 0.2)
                elif t % 400 == 100:
                    o.arr('xfrc_applied')[:] = 0
                o.step_pd(u)
                if (t + 1) % 100 == 0:
                    want.append(o.arr('qpos')[:o.nq].copy())
            err[j] = float(np.abs(got[:, j, :] - np.array(want)).max())
            o.close()
        med, p90, worst = float(np.median(err)), float(np.percentile(err, 90)), float(err.max())
        print('4096 fp32 with device-row pushes: median %.1e, p90 %.1e, worst %.1e' % (med, p90, worst))
        assert med <= BARS[3][0] and p90 <= BARS[3][1] and worst <= BARS[3][2], (med, p90, worst)
        assert int(b.counters()[:, 4].sum()) == 0
        assert b.device_ptr('contact') is None or not b.device_ptr('contact')   # the plain twin: no carried rows
        b.close()
    finally:
        if old is not None:
            os.environ['CASSIE_B200_DEBUG'] = old


def _rand(b, seed):
    rng = np.random.default_rng(seed)
    nb = b.L.cassie_batch_nbody(b.h)
    return rng.normal(size=(b.n, nb, 6)) * 5, rng.normal(size=(b.n, b.nv))


def test_verbs(P):
    """masked set / get round trip with NULL parts kept; validation; reset zeroes the rows; clear_forces keeps qfrc; enable(0) drops them"""
    b = P.CassieBatch(4, modelfile=P.model_path('cassie'), precision=P.FP64)
    z = b.applied_forces()
    assert not np.any(z['xfrc']) and not np.any(z['qfrc'])   # no rows: zeros
    x, q = _rand(b, 1)
    b.set_applied_forces(x, q)
    x2, q2 = _rand(b, 2)
    m = np.array([1, 0, 1, 0], np.uint8)
    b.set_applied_forces(xfrc=x2, mask=m)   # qfrc kept
    got = b.applied_forces()
    assert np.array_equal(got['xfrc'], np.where(m[:, None, None] == 1, x2, x)) and np.array_equal(got['qfrc'], q)
    bad = x2.copy()
    bad[2, 9, 4] = np.nan
    with pytest.raises(RuntimeError, match=r'environment 2, body left-tarsus: xfrc_applied\[4\] is not finite'):
        b.set_applied_forces(xfrc=bad, qfrc=q2)
    badq = q2.copy()
    badq[1, 7] = np.inf
    with pytest.raises(RuntimeError, match='environment 1, dof 7: qfrc_applied is not finite'):
        b.set_applied_forces(qfrc=badq)
    assert np.array_equal(b.applied_forces()['qfrc'], q)   # nothing changed
    b.set_applied_forces(np.zeros_like(x) + x[0, 0])   # the world body too: accepted
    b.clear_forces()
    got = b.applied_forces()
    assert not np.any(got['xfrc']) and np.array_equal(got['qfrc'], q)
    b.set_applied_forces(x, q)
    b.reset(np.array([0, 1, 0, 0], np.uint8))
    got = b.applied_forces()
    assert not np.any(got['xfrc'][1]) and not np.any(got['qfrc'][1]) and np.array_equal(got['qfrc'][0], q[0])
    b.reset()
    got = b.applied_forces()
    assert not np.any(got['xfrc']) and not np.any(got['qfrc'])
    b.enable_applied_forces(False)
    assert not b.device_ptr('applied')
    b.close()


def _run(b, ticks):
    out = []
    for _ in range(ticks):
        b.step(1)
        out.append(b.qpos())
    return np.array(out)


def test_snapshots(P):
    """restore (unmasked and masked) and continue == the undisturbed run, bitwise; a snapshot with rows allocates rows in a batch without them, one
    without rows zeroes the restored environments' rows"""
    b = P.CassieBatch(4, modelfile=P.model_path('cassie'), precision=P.FP64)
    _pd(P, b, 4)
    b.reset()
    x, q = _rand(b, 3)
    b.set_applied_forces(x, q)
    b.step(20)
    s = b.get_state()
    ref = _run(b, 60)
    b.set_applied_forces(*_rand(b, 4))
    b.step(10)
    b.set_state(s)
    assert np.array_equal(_run(b, 60), ref)
    b.set_applied_forces(*_rand(b, 5))
    b.step(10)
    m = np.array([0, 1, 1, 0], np.uint8)
    before = b.applied_forces()
    b.set_state(s, mask=m)
    got = b.applied_forces()
    assert np.array_equal(got['qfrc'][1:3], q[1:3]) and np.array_equal(got['qfrc'][0], before['qfrc'][0])
    c = P.CassieBatch(4, modelfile=P.model_path('cassie'), precision=P.FP64)
    _pd(P, c, 4)
    c.set_state(s)   # rows come with the snapshot
    assert np.array_equal(c.applied_forces()['qfrc'], q)
    assert np.array_equal(_run(c, 60), ref)
    c.enable_applied_forces(False)
    s0 = c.get_state()   # without rows
    b.set_state(s0, mask=np.array([1, 0, 0, 0], np.uint8))
    got = b.applied_forces()
    assert not np.any(got['qfrc'][0]) and not np.any(got['xfrc'][0]) and np.any(got['qfrc'][1])
    b.free_state(s)
    c.free_state(s0)
    b.close()
    c.close()


def test_device_row_write_equals_verb_write(P):
    """a write through torch_view('applied') equals the same values through the verb, bit for bit"""
    import torch
    out = []
    for how in ('verb', 'view'):
        b = P.CassieBatch(8, modelfile=P.model_path('cassie_tray_box'), precision=P.FP32)
        _pd(P, b, 8)
        b.reset()
        x, q = _rand(b, 6)
        x[:, :, :] *= 0.1
        q *= 0.1
        if how == 'verb':
            b.set_applied_forces(x, q)
        else:
            b.enable_applied_forces()
            v = b.torch_view('applied')
            row = np.zeros((8, 232), np.float32)
            row[:, :x.shape[1] * 6] = x.reshape(8, -1)
            row[:, 192:192 + b.nv] = q
            v.copy_(torch.as_tensor(row, device='cuda'))
            torch.cuda.synchronize()
        out.append(_run(b, 50))
        b.close()
    assert np.array_equal(out[0], out[1])


def test_legacy_simulator(P, oracle_mod):
    """cassie_sim_qfrc writes follow the oracle's qfrc_applied; cassie_sim_copy, cassie_get_state / cassie_set_state carry the rows;
    cassie_sim_step_pd_batch with rows equals the compact path bit for bit"""
    L = P.lib()
    L.cassie_sim_qfrc.restype = C.POINTER(C.c_double)
    L.cassie_sim_qfrc.argtypes = [C.c_void_p]
    s = P.CassieSim(P.model_path('cassie'))
    o = oracle_mod.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    qf = L.cassie_sim_qfrc(s.c)
    rng = np.random.default_rng(9)
    val = rng.normal(size=32) * 2
    for i in range(32):
        qf[i] = val[i]
    o.arr('qfrc_applied')[:] = val
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    pd = P.pd_in_t()
    for side, leg in enumerate((pd.leftLeg, pd.rightLeg)):
        for i in range(5):
            leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
    for _ in range(200):
        s.step_pd(pd)
        o.step_pd(u)
    assert np.abs(s.qpos()[:35] - o.arr('qpos')).max() < 1e-9
    assert np.array_equal(np.array(qf[:32]), val)   # the mirror holds what the rows hold
    st = s.get_state()
    d = s.duplicate()   # cassie_sim_copy
    s2 = P.CassieSim(P.model_path('cassie'))
    s2.set_state(st)
    for _ in range(50):
        s.step_pd(pd)
        d.step_pd(pd)
        s2.step_pd(pd)
    assert np.array_equal(s.qpos(), d.qpos()) and np.array_equal(s.qpos(), s2.qpos())
    # the AoS entry point with rows == the compact path
    b1 = P.CassieBatch(4, modelfile=P.model_path('cassie'), precision=P.FP64)
    b2 = P.CassieBatch(4, modelfile=P.model_path('cassie'), precision=P.FP64)
    x, q = _rand(b1, 10)
    for bb in (b1, b2):
        bb.set_applied_forces(x * 0.5, q * 0.5)
    pin = (P.pd_in_t * 4)(*[pd] * 4)
    _pd(P, b2, 4)
    for _ in range(50):
        b1.step_pd(pin)
        b2.step(1)
    assert np.array_equal(b1.qpos(), b2.qpos())
    for x_ in (s, d, s2):
        x_.close() if hasattr(x_, 'close') else None
    b1.close()
    b2.close()
    o.close()
