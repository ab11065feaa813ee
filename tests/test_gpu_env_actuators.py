"""GPU: per-environment actuators (cassie_batch_set_env_actuators, the F_AC instances), the batched actuator state and the legacy verbs on it, against
the fp64 oracle given the same ctrlrange, rpm and delay (tests/actuator_support.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from actuator_support import LINE, NU, ActOracle, pd_row, saturating_pd, table
from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_gpu_aos_parity import Fields, _rel

pytestmark = pytest.mark.gpu
OB_MTORQUE = 20


@pytest.fixture(scope='module')
def P():
    """batches of this module run without the stage dumps, whatever an earlier module left in the environment"""
    old = os.environ.pop('CASSIE_B200_DEBUG', None)
    yield product()
    if old is not None:
        os.environ['CASSIE_B200_DEBUG'] = old


def to_pin(P, u):
    """the oracle's pd_in_t as the product's (the same C struct)"""
    p = P.pd_in_t()
    C.memmove(C.addressof(p), C.addressof(u), C.sizeof(p))
    return p


def batch_pd(P, u, n):
    """the batch's PD rows [n, PD_WIDTH] holding a pd_in_t's motorPd branch in every environment"""
    rows = np.zeros((n, P.PD_WIDTH))
    rows[:, :50] = pd_row(u)
    return rows


def four_setups(model='cassie'):
    """(ctrlrange [4, nu, 2], rpm [4, nu], delay [4, nu]): d = 0; d = 3 with hi at 60 % and an asymmetric range, lo = -0.3 hi (the actuation's lower
    clamp acts); d = 6 with rpm at 70 %; the model's values"""
    _, cr, rpm = table(model)
    crs, rpms, dls = np.stack([cr] * 4), np.stack([rpm] * 4), np.array([[0] * NU, [3] * NU, [6] * NU, [6] * NU])
    crs[1, :, 1] *= 0.6
    crs[1, :, 0] = -0.3 * crs[1, :, 1]
    rpms[2] *= 0.7
    return crs, rpms, dls


def run_compact(P, O, b, n, T):
    """T single-tick calls of saturating inputs; per call qpos, drive torques and PGS iteration counts"""
    qs, ts, its = [], [], []
    for k in range(T):
        b.set_pd(batch_pd(P, saturating_pd(O, k), n))
        b.step(1)
        qs.append(b.qpos())
        ts.append(b.obs()[:, OB_MTORQUE:OB_MTORQUE + NU])
        its.append(b.counters()[:, 3].copy())
    return np.array(qs), np.array(ts), np.array(its)


def test_four_envs_fp64_follow_their_oracles(P, oracle_mod):
    """four fp64 environments, each against its own oracle over 1000 ticks: qpos <= 1e-9, drive torques <= 1e-9, equal PGS iteration counts"""
    O, n, T = oracle_mod, 4, 1000
    crs, rpms, dls = four_setups()
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_env_actuators(crs, rpms, dls)
    cr, rp, dl = b.env_actuators()
    assert np.array_equal(cr, crs) and np.array_equal(rp, rpms) and np.array_equal(dl, dls)
    qs, ts, its = run_compact(P, O, b, n, T)
    assert int(b.counters()[:, 4].sum()) == 0
    for e in range(n):
        o = ActOracle(O, 'cassie', crs[e], rpms[e], dls[e])
        wq, wt, same, below = 0.0, 0.0, True, 0
        for k in range(T):
            o.step_pd(saturating_pd(O, k))
            below += int(np.sum(o.o.arr('ctrl')[:NU] < crs[e, :, 0]))   # ticks at which the actuation clamps ctrl up to lo
            wq = max(wq, np.abs(qs[k, e, :o.o.nq] - o.o.arr('qpos')).max())
            wt = max(wt, np.abs(ts[k, e] - o.drive_torque()).max())
            same = same and int(its[k, e]) == o.o.get_int('solver_iter')
        o.close()
        print('env %d: qpos %.2e, drive torque %.2e, %d motor-ticks clamped at lo' % (e, wq, wt, below))
        assert wq <= 1e-9 and wt <= 1e-9 and same, (e, wq, wt, same)
        assert e != 1 or below > 0   # the asymmetric range's lower bound acted
    b.close()


def test_model_values_equal_the_body_pos_twin(P, oracle_mod):
    """model-valued actuator rows (d1d7) against the same batch with model-valued offset rows only (its F_BP twin d157), 1000 fp64 ticks: <= 1e-12,
    bitwise expected"""
    O, n, T = oracle_mod, 4, 1000
    _, cr, rpm = table('cassie')
    a = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    a.set_env_body_pos(a.env_body_pos())
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_env_actuators(cr, rpm, np.full(NU, LINE))
    assert np.array_equal(b.env_body_pos(), a.env_body_pos())
    qa, ta, _ = run_compact(P, O, a, n, T)
    qb, tb, _ = run_compact(P, O, b, n, T)
    worst = max(np.abs(qa - qb).max(), np.abs(ta - tb).max())
    print('model-valued actuator rows vs the F_BP twin: worst %.2e, bitwise %s' % (worst, np.array_equal(qa, qb) and np.array_equal(ta, tb)))
    assert worst <= 1e-12
    a.close()
    b.close()


def test_fp32_4096_random_rows_sampled(P, oracle_mod):
    """4096 fp32 environments with random rows (delay uniform on 0..6, hi x [0.6, 1.2], rpm x [0.7, 1.3]); after 600 standing ticks 64 sampled
    environments against the oracle: median <= 1e-5, p90 <= 1e-4, worst <= 1e-3; no contact dropped"""
    O, n, T = oracle_mod, 4096, 600
    _, cr, rpm = table('cassie')
    rng = np.random.default_rng(31)
    crs = np.broadcast_to(cr, (n, NU, 2)).copy()
    crs[:, :, 1] *= rng.uniform(0.6, 1.2, (n, NU))
    rpms = rpm * rng.uniform(0.7, 1.3, (n, NU))
    dls = rng.integers(0, LINE + 1, (n, NU))
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    b.set_env_actuators(crs, rpms, dls)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.step(T)
    q = b.qpos()
    assert (b.counters()[:, 4] == 0).all()
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    errs = []
    for e in np.random.default_rng(5).choice(n, 64, replace=False):
        o = ActOracle(O, 'cassie', crs[e], rpms[e], dls[e])
        for _ in range(T):
            o.step_pd(u)
        errs.append(np.abs(q[e, :o.o.nq] - o.o.arr('qpos')).max())
        o.close()
    errs = np.array(errs)
    print('fp32 4096 random actuator rows: median %.2e p90 %.2e worst %.2e' % (np.median(errs), np.percentile(errs, 90), errs.max()))
    assert np.median(errs) <= 1e-5 and np.percentile(errs, 90) <= 1e-4 and errs.max() <= 1e-3
    b.close()


def test_aos_path_every_field(P, oracle_mod):
    """cassie_sim_step_pd_batch with actuator rows, 4 fp64 environments over 300 calls: every state_out_t field against the oracle's twin at the fp64
    bars of test_gpu_aos_parity.py (qpos, decoded fields and torques <= 1e-9, velocities 1e-7, filtered fields and forces 1e-8 relative)"""
    O, F, n, T = oracle_mod, Fields(P), 4, 300
    crs, rpms, dls = four_setups()
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_env_actuators(crs, rpms, dls)
    pin = (P.pd_in_t * n)()
    os_ = [ActOracle(O, 'cassie', crs[e], rpms[e], dls[e]) for e in range(n)]
    y = P.state_out_t()
    G, worst = F.group, {'qpos': 0.0}
    for k in range(T):
        u = saturating_pd(O, k)
        for e in range(n):
            C.memmove(C.addressof(pin[e]), C.addressof(u), C.sizeof(u))
        ys = b.step_pd(pin)
        q = b.qpos()
        d = F.doubles(ys, n)
        fl = F.flags(ys, n)
        for e, o in enumerate(os_):
            o.step_pd(u, y)
            wd = F.doubles(y, 1)[0]
            worst['qpos'] = max(worst['qpos'], float(np.abs(q[e, :o.o.nq] - o.o.arr('qpos')).max()))
            for g in ('pos', 'vel', 'torque', 'accel'):
                worst[g] = max(worst.get(g, 0.0), float(np.abs(d[e, G[g]] - wd[G[g]]).max()))
            for g in ('filtered', 'force'):
                worst[g] = max(worst.get(g, 0.0), float(_rel(wd[G[g]], d[e, G[g]]).max()))
            assert np.array_equal(d[e, G['const']], wd[G['const']]) and np.array_equal(fl[e], F.flags(y, 1)[0]), (k, e)
    print('AoS with actuator rows vs oracle: ' + ' '.join('%s %.1e' % kv for kv in worst.items()))
    assert worst['qpos'] <= 1e-9 and worst['pos'] <= 1e-9 and worst['torque'] <= 1e-9 and worst['accel'] <= 1e-9, worst
    assert worst['vel'] <= 1e-7 and worst['filtered'] <= 1e-8 and worst['force'] <= 1e-8, worst
    for o in os_:
        o.close()
    b.close()


def test_actuator_state_round_trip_and_mid_run_writes(P, oracle_mod):
    """get / set round-trip bitwise; a delay line and filter states written mid-run into the batch and into the oracles, then 200 more ticks: <= 1e-9"""
    O, n = oracle_mod, 4
    crs, rpms, dls = four_setups()
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_env_actuators(crs, rpms, dls)
    os_ = [ActOracle(O, 'cassie', crs[e], rpms[e], dls[e]) for e in range(n)]
    for k in range(100):
        b.set_pd(batch_pd(P, saturating_pd(O, k), n))
        b.step(1)
        for o in os_:
            o.step_pd(saturating_pd(O, k))
    s = b.actuator_state()
    for e, o in enumerate(os_):   # the state itself agrees with the oracle's
        assert np.abs(s['torque_delay'][e] - o.line).max() < 1e-9
        assert np.array_equal(s['drive_filter'][e].ravel(), np.ctypeslib.as_array(o.o.L.osim_drive_filter(o.o.h), shape=(90,)))
    b.set_actuator_state(**s)
    s2 = b.actuator_state()
    assert all(np.array_equal(s[k], s2[k]) for k in s)
    rng = np.random.default_rng(3)
    td = s['torque_delay'] + rng.uniform(-0.5, 0.5, s['torque_delay'].shape)
    jx = s['joint_x'] + rng.uniform(-1e-3, 1e-3, s['joint_x'].shape)
    jy = s['joint_y'] + rng.uniform(-1e-2, 1e-2, s['joint_y'].shape)
    df = s['drive_filter'] + rng.integers(-20, 20, s['drive_filter'].shape).astype(np.int32)
    mask = np.array([1, 1, 0, 1], dtype=np.uint8)
    b.set_actuator_state(td, df, jx, jy, mask=mask)
    s3 = b.actuator_state()
    assert np.array_equal(s3['torque_delay'][2], s['torque_delay'][2]) and np.array_equal(s3['torque_delay'][0], td[0])
    L = os_[0].o.L
    for e, o in enumerate(os_):
        if not mask[e]:
            continue
        o.line[:] = td[e]
        np.ctypeslib.as_array(L.osim_drive_filter(o.o.h), shape=(90,))[:] = df[e].ravel()
        np.ctypeslib.as_array(L.osim_joint_filter_x(o.o.h), shape=(24,))[:] = jx[e].ravel()
        np.ctypeslib.as_array(L.osim_joint_filter_y(o.o.h), shape=(18,))[:] = jy[e].ravel()
    worst = 0.0
    for k in range(100, 300):
        b.set_pd(batch_pd(P, saturating_pd(O, k), n))
        b.step(1)
        q, t = b.qpos(), b.obs()[:, OB_MTORQUE:OB_MTORQUE + NU]
        for e, o in enumerate(os_):
            o.step_pd(saturating_pd(O, k))
            worst = max(worst, np.abs(q[e, :o.o.nq] - o.o.arr('qpos')).max(), np.abs(t[e] - o.drive_torque()).max())
    print('after mid-run state writes: worst %.2e' % worst)
    assert worst <= 1e-9
    for o in os_:
        o.close()
    b.close()


def test_legacy_verbs_against_the_oracle(P, oracle_mod):
    """the eight legacy verbs through a cassie_sim_t agree with the oracle's delay line and filters; ctrl is the applied control, writes through it do
    not reach the next step, and it reads zeros after full_reset"""
    O = oracle_mod
    s = P.CassieSim(P.model_path('cassie'))
    o = ActOracle(O, 'cassie')
    for k in range(150):
        u = saturating_pd(O, k)
        s.step_pd(to_pin(P, u))
        o.step_pd(u)
    L = o.o.L
    assert np.abs(s.get_torque_delay() - o.line).max() < 1e-9
    jf = s.get_joint_filter()
    ox, oy = np.ctypeslib.as_array(L.osim_joint_filter_x(o.o.h), shape=(6, 4)), np.ctypeslib.as_array(L.osim_joint_filter_y(o.o.h), shape=(6, 3))
    assert max(np.abs(np.array(jf[j].x[:]) - ox[j]).max() for j in range(6)) < 1e-9
    assert max(np.abs(np.array(jf[j].y[:]) - oy[j]).max() for j in range(6)) < 1e-9
    dfp = s.get_drive_filter()
    od = np.ctypeslib.as_array(L.osim_drive_filter(o.o.h), shape=(10, 9))
    assert all(list(dfp[i].x[:]) == list(od[i]) for i in range(10))
    ctrl = np.array(s.ctrl())
    assert np.allclose(ctrl, o.o.arr('ctrl')[:NU], rtol=3e-16, atol=0), ctrl - o.o.arr('ctrl')[:NU]   # the drive torque over the gear: 1 ulp
    # writes: the delay line and both filters through the set verbs and the borrowed mirrors, into the oracle too; ctrl writes change nothing
    rng = np.random.default_rng(8)
    td = o.line + rng.uniform(-0.3, 0.3, (10, 6))
    s.set_torque_delay(td)
    o.line[:] = td
    x, y = ox + 1e-3, oy + 1e-2
    s.set_joint_filter(x.ravel(), y.ravel())
    ox[:], oy[:] = x, y
    dfp = s.get_drive_filter()
    for i in range(10):
        dfp[i].x[0] += 7
    od[:, 0] += 7
    jf = s.get_joint_filter()
    jf[2].y[1] += 0.05
    oy[2, 1] += 0.05
    s.set_ctrl([100.0] * NU)
    worst = 0.0
    for k in range(150, 300):
        u = saturating_pd(O, k)
        s.step_pd(to_pin(P, u))
        o.step_pd(u)
        worst = max(worst, np.abs(s.qpos() - o.o.arr('qpos')[:35]).max())
    print('legacy actuator verbs after writes: worst qpos %.2e' % worst)
    assert worst <= 1e-9
    di = np.zeros(90, dtype=np.int32)
    s.L.cassie_sim_get_drive_filter(s.c, di.ctypes.data_as(C.POINTER(C.c_int)))
    assert np.array_equal(di, od.ravel())
    s.set_drive_filter(od.ravel())
    s.full_reset()
    assert np.array_equal(np.array(s.ctrl()), np.zeros(NU)) and np.array_equal(s.get_torque_delay(), np.zeros((10, 6)))
    o.close()


def test_lifecycle(P, oracle_mod):
    """reset and masked set_state leave the rows alone; clear returns to what ran before (bitwise a batch that never had rows); the implicit offset
    rows: get reports the model's, clear_env_body_pos keeps them holding the model's, clear_env_actuators drops them unless a body-offset call wrote
    them since"""
    O, n = oracle_mod, 4
    crs, rpms, dls = four_setups()
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    ref = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    bp0 = ref.env_body_pos()
    b.set_env_actuators(crs, rpms, dls)
    assert np.array_equal(b.env_body_pos(), bp0)
    rows0 = b.torch_view('actuators').cpu().numpy().copy()   # what the kernels read
    snap = b.get_state()
    b.reset()
    b.step(20)
    b.set_state(snap, mask=np.array([1, 0, 1, 0], dtype=np.uint8))
    b.sync()
    assert np.array_equal(b.torch_view('actuators').cpu().numpy(), rows0)
    cr, rp, dl = b.env_actuators()
    assert np.array_equal(cr, crs) and np.array_equal(rp, rpms) and np.array_equal(dl, dls)
    with pytest.raises(RuntimeError):
        bad = dls.copy(); bad[3, 4] = 7
        b.set_env_actuators(delay=bad)
    with pytest.raises(RuntimeError):
        bad = crs.copy(); bad[0, 1] = [1.0, -1.0]
        b.set_env_actuators(ctrlrange=bad)
    assert all(np.array_equal(x, y) for x, y in zip(b.env_actuators(), (crs, rpms, dls)))
    dev = b.torch_view('actuators')
    assert tuple(dev.shape) == (n, 40)
    b.clear_env_body_pos()   # keeps the offset rows (model values) while actuator rows are there
    assert np.array_equal(b.env_body_pos(), bp0)
    b.clear_env_actuators()
    assert b.device_ptr('actuators') is None or not b.device_ptr('actuators')
    # set-then-clear is bitwise a batch that never had rows
    b.reset()
    ref.reset()
    for x in (b, ref):
        x.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        x.step(50)
    assert np.array_equal(b.qpos(), ref.qpos()) and np.array_equal(b.obs(), ref.obs())
    # offsets written after the actuator rows stay when the actuator rows go
    bp = bp0.copy()
    bp[:, 1] += [0.0, 0.0, 0.01]
    b.set_env_actuators(crs, rpms, dls)
    b.set_env_body_pos(bp)
    b.clear_env_actuators()
    assert np.array_equal(b.env_body_pos(), bp)
    b.close()
    ref.close()


def _rows(P, L, bh, n):
    """a torch view [n, ACT_W] of a batch handle's actuator rows (fp64)"""
    import torch
    L.cassie_batch_device_ptr.restype = C.c_void_p
    L.cassie_batch_device_ptr.argtypes = [C.c_void_p, C.c_char_p]
    ptr = L.cassie_batch_device_ptr(bh, b'actuators')
    assert ptr

    class _A:
        pass
    a = _A()
    a.__cuda_array_interface__ = dict(shape=(n, 40), typestr='<f8', data=(ptr, False), version=2)
    return torch.as_tensor(a, device='cuda')


def test_device_written_rows_are_what_the_verbs_work_on(P, oracle_mod):
    """rows written through torch_view('actuators') survive a masked set_env_actuators (of the delay only) in the unmasked environments, get reports
    them, and cassie_sim_copy copies the rows as they are: the copy then steps bit for bit as its source"""
    import torch
    O, n = oracle_mod, 4
    crs, rpms, dls = four_setups()
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_env_actuators(crs, rpms, dls)
    v = b.torch_view('actuators')
    v[2, 10:20] *= 0.8        # hi
    v[2, 20:30] *= 0.9        # wmax
    v[2, 30:40] = 1.0         # delay
    v[3, 30:40] = float('nan')   # read as 0 by the kernel
    torch.cuda.synchronize()
    before = v.cpu().numpy().copy()
    b.set_env_actuators(delay=np.full((n, NU), 4), mask=np.array([1, 0, 0, 0], dtype=np.uint8))
    after = v.cpu().numpy()
    assert np.array_equal(after[1:], before[1:], equal_nan=True)
    assert np.array_equal(after[0, :30], before[0, :30]) and np.all(after[0, 30:] == 4)
    cr, rp, dl = b.env_actuators()
    assert np.all(dl[0] == 4) and np.all(dl[2] == 1) and np.all(dl[3] == 0) and np.array_equal(dl[1], dls[1])
    assert np.array_equal(cr[2, :, 1], before[2, 10:20]) and np.array_equal(cr[2, :, 0], crs[2, :, 0]) and np.array_equal(cr[1], crs[1])
    assert np.allclose(rp[2], before[2, 20:30] * 60 / (2 * np.pi), rtol=1e-15, atol=0) and np.array_equal(rp[1], rpms[1])
    # the environments run with what get reports: environment 2 against an oracle given it
    o = ActOracle(O, 'cassie', cr[2], rp[2], dl[2])
    for k in range(200):
        b.set_pd(batch_pd(P, saturating_pd(O, k), n))
        b.step(1)
        o.step_pd(saturating_pd(O, k))
    assert np.abs(b.qpos()[2, :o.o.nq] - o.o.arr('qpos')).max() <= 1e-9
    o.close()
    b.close()
    # cassie_sim_copy: rows set on a simulator's batch and then written on the device are copied as the rows hold them
    L = P.lib()
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    L.cassie_batch_set_env_actuators.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int), C.c_void_p]
    L.cassie_batch_set_env_actuators.restype = C.c_int
    s1, s2 = P.CassieSim(P.model_path('cassie')), P.CassieSim(P.model_path('cassie'))
    b1 = L.cassie_sim_batch(s1.c)
    c1 = np.ascontiguousarray(crs[1])
    r1 = np.ascontiguousarray(rpms[2])
    d1 = np.ascontiguousarray(np.full(NU, 2, dtype=np.int32))
    assert L.cassie_batch_set_env_actuators(b1, c1.ctypes.data_as(C.POINTER(C.c_double)), r1.ctypes.data_as(C.POINTER(C.c_double)), d1.ctypes.data_as(C.POINTER(C.c_int)), None) == 0
    w = _rows(P, L, b1, 1)
    w[0, 30:35] = 5.0
    torch.cuda.synchronize()
    for k in range(30):
        s1.step_pd(to_pin(P, saturating_pd(O, k)))
    s2.copy(s1)
    b2 = L.cassie_sim_batch(s2.c)
    assert np.array_equal(_rows(P, L, b2, 1).cpu().numpy(), w.cpu().numpy())
    for k in range(30, 230):
        u = to_pin(P, saturating_pd(O, k))
        s1.step_pd(u)
        s2.step_pd(u)
    assert np.array_equal(s1.qpos(), s2.qpos())
