"""GPU: per-environment mechanics (cassie_batch_set_env_mechanics, the F_MC instances: link inertia, rotor armature, hinge springs), against the fp64
oracle given the same body_inertia, dof_armature, jnt_stiffness and qpos_spring (a temporary copy of its model table, tests/mechanics_support.py)."""
import ctypes as C

import numpy as np
import pytest

from actuator_support import NU, pd_row, saturating_pd
from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product
from mechanics_support import HINGE, changeable_bodies, oracle_with, random_mechanics, table
from test_accelerations import oracle_row, split
from test_dynamics import full_m
from test_frames import CFRC, VEL, all_frames, omodel, oracle_frames

pytestmark = pytest.mark.gpu
PARTS = ('inertia', 'armature', 'stiffness', 'springref')
MC_STIFF, MC_SPRING = 128, 160


@pytest.fixture(scope='module')
def P():
    return product()


def base(b):
    """the model's values as the batch reports them without rows (inertia, armature, stiffness, springref)"""
    m = b.env_mechanics()
    return [m[k][0] for k in PARTS]


def batch_values(model, n, seed, b0):
    """[n, ...] per part: environment e gets random_mechanics(model, seed + e) from the batch's model values; environment 0 the model's"""
    vals = [b0] + [random_mechanics(model, seed + e, b0) for e in range(1, n)]
    return [np.stack([v[p] for v in vals]) for p in range(4)]


def oracle_for(O, model, vals, e, **kw):
    return oracle_with(O, model, *[v[e] for v in vals], **kw)


def test_four_envs_fp64_with_set_const(P, oracle_mod):
    """4 environments, each its own mechanics, one also its own masses == 4 oracles with the same tables; a masked set_const with state reset on two of
    them (each against its oracle's mj_setConst with the same inertia and armature), then 250 more ticks: qpos within 1e-9, equal PGS iteration counts"""
    O, n, model = oracle_mod, 4, 'cassie'
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    vals = batch_values(model, n, 40, base(b))
    b.set_env_mechanics(*vals)
    got = b.env_mechanics()
    assert all(np.array_equal(got[k], v) for k, v in zip(PARTS, vals))
    mass = b.get_model('body_mass')
    mass[2] *= 1.1
    b.set_model('body_mass', mass)
    os_ = [oracle_for(O, model, vals, e, **({'body_mass': mass[e]} if e == 2 else {})) for e in range(n)]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    for o in os_:
        o.forward()
    b.reset()

    def run(T):
        same = True
        for _ in range(T):
            b.step(1)
            it = b.counters()[:, 3]
            for e, o in enumerate(os_):
                o.step_pd(u)
                same = same and int(it[e]) == o.get_int('solver_iter')
        q = b.qpos()
        return [float(np.abs(q[e, :o.nq] - o.arr('qpos')).max()) for e, o in enumerate(os_)], same

    w, same = run(250)
    print('before set_const: ' + ' '.join('%.1e' % x for x in w))
    assert max(w) < 1e-9 and same, (w, same)
    mask = np.array([0, 1, 0, 1], dtype=np.uint8)
    before = b.qpos()
    b.set_const(mask, reset_state=True)
    assert np.array_equal(b.qpos()[[0, 2]], before[[0, 2]])
    for i in (1, 3):
        os_[i].set_const()
    w, same = run(250)
    print('after set_const: ' + ' '.join('%.1e' % x for x in w))
    assert max(w) < 1e-9 and same, (w, same)
    assert np.abs(b.qpos()[1] - b.qpos()[0]).max() > 1e-5   # the values moved the environments apart
    for o in os_:
        o.close()
    b.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_mass'])
def test_fp32_4096_sampled_against_the_oracle(P, oracle_mod, model):
    """4096 fp32 environments with seeded mechanics; 64 sampled environments replayed in the oracle for 600 ticks.  Bars over the sample's worst qpos
    error (DESIGN.md section 3): median <= 1e-5, p90 <= 3e-5, worst <= 1e-3; no contact dropped"""
    n, T = 4096, 600
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32)
    b0 = base(b)
    vals = batch_values(model, n, 1000, b0)
    b.set_env_mechanics(*vals)
    b.reset()
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.step(T)
    q = b.qpos()
    assert (b.counters()[:, 4] == 0).all()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    errs = []
    for e in np.random.default_rng(5).choice(n, 64, replace=False):
        o = oracle_for(oracle_mod, model, vals, e)
        o.forward()
        for _ in range(T):
            o.step_pd(u)
        errs.append(np.abs(q[e, :o.nq] - o.arr('qpos')).max())
        o.close()
    errs = np.array(errs)
    print(model, 'median %.2e p90 %.2e worst %.2e' % (np.median(errs), np.percentile(errs, 90), errs.max()))
    assert np.median(errs) <= 1e-5 and np.percentile(errs, 90) <= 3e-5 and errs.max() <= 1e-3
    b.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_launch_modes_follow_the_oracle(P, oracle_mod, fp32):
    """dynamics rows (M's diagonal carries the armature and the link inertias), frames (every body) and acceleration rows with mechanics rows (d11d7,
    f11d7) against oracles with the same tables stepped alongside, at the tolerances of test_gpu_env_body_pos.py: fp64 frame poses within 1e-10,
    velocities and contact forces within 1e-8, qacc within 1e-8 of its largest magnitude, M within 1e-12 of its largest entry; fp32 frame poses within
    1e-3 and M within 1e-5 (at the batch's own state)"""
    n, model, ticks = 3, 'cassie', 200
    m = omodel(model)
    names, kinds = all_frames(model)
    nbn = len(m['names_body'])
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32 if fp32 else P.FP64)
    vals = batch_values(model, n, 60, base(b))
    b.set_env_mechanics(*vals)
    b.set_frames(names[:nbn], kinds[:nbn])
    b.enable_accelerations()
    b.reset()
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    os_ = [oracle_for(oracle_mod, model, vals, e) for e in range(n)]
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for o in os_:
        o.forward()
    for _ in range(ticks):
        b.step(1)
        for o in os_:
            o.step_pd(u)
    fr, qa = b.frames(), b.qacc()
    q, v = b.qpos(), b.qvel()
    b.compute_dynamics()
    M = b.dynamics()['M']
    for e, o in enumerate(os_):
        want = oracle_frames(o, m, names[:nbn], kinds[:nbn])
        dpos = np.abs(fr[e, :, :VEL] - want[:, :VEL]).max()
        d = oracle_for(oracle_mod, model, vals, e)   # M at the batch's own state
        d.arr('qpos')[:] = q[e, :d.nq]
        d.arr('qvel')[:] = v[e, :d.nv]
        d.forward()
        wM = full_m(d.arr('qM'), m)
        dM = np.abs(M[e][:d.nv, :d.nv] - wM).max() / np.abs(wM).max()
        d.close()
        if fp32:
            assert dpos <= 1e-3 and dM <= 1e-5, (e, dpos, dM)
            continue
        wq = split(oracle_row(o, m, names[:nbn], kinds[:nbn]), nbn)[0]
        assert dpos <= 1e-10 and dM <= 1e-12, (e, dpos, dM)
        assert np.abs(fr[e, :, VEL:CFRC] - want[:, VEL:CFRC]).max() <= 1e-8 and np.abs(fr[e, :, CFRC:] - want[:, CFRC:]).max() <= 1e-8, e
        assert np.abs(qa[e] - wq[:b.nv]).max() <= 1e-8 * np.abs(wq).max(), e
    # the armature is on M's diagonal: environments 1 and 2 differ from 0 there by at least their armature difference at a motor dof
    dg = np.array([np.diag(M[e][:32, :32]) for e in range(n)])
    assert np.abs(dg[1, 6] - dg[0, 6]) > 0.5 * np.abs(vals[1][1, 6] - vals[1][0, 6])
    for o in os_:
        o.close()
    b.close()


def _steady(P, b, n, T, O=None):
    rows = []
    for k in range(T):
        b.set_pd(np.tile(np.concatenate([pd_row(saturating_pd(O, k)), np.zeros(P.PD_WIDTH - 50)]), (n, 1)))
        b.step(1)
    return [x.copy() for x in (b.qpos(), b.qvel(), b.obs(), b.aux(), b.counters())]


@pytest.mark.parametrize('fp32', [False, True])
def test_model_rows_are_bitwise_the_actuator_twin(P, oracle_mod, fp32):
    """model-valued mechanics rows (f11d7 / d11d7) against the same batch with model-valued actuator rows only (their F_AC twins f1d7 / d1d7) over 1000
    saturating ticks: qpos, qvel, obs, aux and the counters bit for bit"""
    n, prec = 64, (P.FP32 if fp32 else P.FP64)
    a, b = (P.CassieBatch(n, precision=prec) for _ in range(2))
    for x in (a, b):
        x.enable_aux()
    a.set_env_actuators(*a.env_actuators())
    b.set_env_mechanics(*base(b))
    ra, rb = _steady(P, a, n, 1000, oracle_mod), _steady(P, b, n, 1000, oracle_mod)
    for name, x, y in zip(('qpos', 'qvel', 'obs', 'aux', 'counters'), ra, rb):
        assert np.array_equal(x, y), name
    a.close()
    b.close()


def test_aos_entry_point_equals_compact_path(P):
    """cassie_sim_step_pd_batch with mechanics rows == the compact path with the same rows and inputs, bit for bit"""
    n = 4096
    a, b = P.CassieBatch(n, precision=P.FP32), P.CassieBatch(n, precision=P.FP32)
    vals = batch_values('cassie', n, 300, base(a))
    for x in (a, b):
        x.set_env_mechanics(*vals)
    b.enable_estimator_device(True)
    pd = (P.pd_in_t * n)()
    for e in range(n):
        for side, leg in enumerate((pd[e].leftLeg, pd[e].rightLeg)):
            for i in range(5):
                leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    for _ in range(200):
        a.step_pd(pd)
        b.step(1)
    assert np.array_equal(a.qpos(), b.qpos()) and np.array_equal(a.obs(), b.obs())
    a.close()
    b.close()


def test_rows_are_model_inputs(P, oracle_mod):
    """refusals change nothing; reset and snapshot restore keep the rows; the implicit actuator rows; a device-pointer write takes effect at the next
    launch and get reports it; clear returns bitwise to a batch that never had rows"""
    import torch
    model, n = 'cassie_tray_box', 4
    t = table(model)
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    ref = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    b0 = base(b)
    ac0 = b.env_actuators()
    vals = batch_values(model, n, 20, b0)
    b.set_env_mechanics(*vals)
    assert all(np.array_equal(x, y) for x, y in zip(b.env_actuators(), ac0))   # implicit actuator rows hold the model's
    nb = len(t['body_weldid'])
    hinge = [j for j in range(len(t['jnt_type'])) if t['jnt_type'][j] == HINGE]
    slide = [j for j in range(len(t['jnt_type'])) if t['jnt_type'][j] == 2]
    for part, idx, v in ((0, (2, 0, 0), 1.0), (0, (1, nb - 1, 0), 1.0), (1, (3, 33), 0.5), (1, (0, 6), -1.0), (2, (1, slide[0]), 1e5), (3, (2, slide[1]), 0.3),
                         (2, (3, hinge[2]), np.nan), (0, (1, changeable_bodies(model)[0], 2), 1e3)):
        bad = [x.copy() for x in vals]
        bad[part][idx] = v
        with pytest.raises(RuntimeError):
            b.set_env_mechanics(*bad)
    got = b.env_mechanics()
    assert all(np.array_equal(got[k], x) for k, x in zip(PARTS, vals))
    b.step(50)
    s = b.get_state()
    b.reset()
    b.set_state(s, mask=np.array([1, 0, 1, 0], dtype=np.uint8))
    got = b.env_mechanics()
    assert all(np.array_equal(got[k], x) for k, x in zip(PARTS, vals))
    # a device write: a stiffer left shin spring in environment 3, seen by get and by the next launch (against an oracle given it)
    dev = b.torch_view('mechanics')
    assert tuple(dev.shape) == (n, 192)
    shin = t['names_joint'].index('left-shin')
    d = t['jnt_dofadr'][shin]
    dev[3, MC_STIFF + d] = 2000.0
    dev[3, MC_SPRING + d] = 0.01
    torch.cuda.synchronize()
    got = b.env_mechanics()
    assert got['stiffness'][3, shin] == 2000.0 and got['springref'][3, shin] == 0.01
    b.reset()
    o = oracle_with(oracle_mod, model, *[got[k][3] for k in PARTS])
    o.forward()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    for _ in range(200):
        b.step(1)
        o.step_pd(u)
    assert np.abs(b.qpos()[3, :o.nq] - o.arr('qpos')).max() <= 1e-9
    o.close()
    # a masked set of one part reads the device rows back: environment 3 keeps its written spring
    b.set_env_mechanics(armature=vals[1], mask=np.array([1, 0, 0, 0], dtype=np.uint8))
    assert b.env_mechanics()['stiffness'][3, shin] == 2000.0
    # clear: back to the model's values and to a batch that never had rows, bitwise
    b.clear_env_mechanics()
    assert not b.device_ptr('mechanics') and not b.device_ptr('actuators')
    got = b.env_mechanics()
    assert all(np.array_equal(got[k][0], x) for k, x in zip(PARTS, b0))
    for x in (b, ref):
        x.reset()
        x.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        x.step(50)
    assert np.array_equal(b.qpos(), ref.qpos()) and np.array_equal(b.obs(), ref.obs())
    # actuator rows written after the mechanics rows stay when the mechanics rows go; clear_env_actuators keeps model-valued rows under mechanics rows
    b.set_env_mechanics(*vals)
    cr = ac0[0].copy()
    cr[:, :, 1] *= 0.9
    b.set_env_actuators(ctrlrange=cr)
    b.clear_env_mechanics()
    assert np.array_equal(b.env_actuators()[0], cr)
    b.clear_env_actuators()
    b.set_env_mechanics(*vals)
    b.clear_env_actuators()
    assert b.device_ptr('actuators') and all(np.array_equal(x, y) for x, y in zip(b.env_actuators(), ac0))
    b.clear_env_mechanics()
    assert not b.device_ptr('actuators')
    b.close()
    ref.close()


def _sim_batch(P):
    L = P.lib()
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    dp = C.POINTER(C.c_double)
    L.cassie_batch_set_env_mechanics.argtypes = [C.c_void_p, dp, dp, dp, dp, C.c_void_p]
    L.cassie_batch_set_env_mechanics.restype = C.c_int
    return L


def _set_sim(L, s, vals):
    arr = [np.ascontiguousarray(v, dtype=np.float64) for v in vals]
    assert L.cassie_batch_set_env_mechanics(L.cassie_sim_batch(s.c), *[a.ctypes.data_as(C.POINTER(C.c_double)) for a in arr], None) == 0


def test_legacy_simulator_copy_and_hold(P, oracle_mod):
    """rows set on a simulator's batch: cassie_sim_step_pd follows the oracle with them, cassie_sim_copy copies them (the copy steps bit for bit as its
    source), and cassie_sim_hold pins the pelvis as it does without rows, also with 0 written into the slide dofs' stiffness slots"""
    import torch
    O = oracle_mod
    L = _sim_batch(P)
    s1, s2, s0 = (P.CassieSim(P.model_path('cassie')) for _ in range(3))
    probe = P.CassieBatch(1, modelfile=P.model_path('cassie'), precision=P.FP64)
    vals = random_mechanics('cassie', 5, base(probe))
    probe.close()
    _set_sim(L, s1, [v[None] for v in vals])
    o = oracle_with(O, 'cassie', *vals)
    pin = P.pd_in_t()
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    C.memmove(C.addressof(pin), C.addressof(u), C.sizeof(pin))
    for _ in range(100):
        s1.step_pd(pin)
        o.step_pd(u)
    assert np.abs(s1.qpos() - o.arr('qpos')[:35]).max() <= 1e-9
    o.close()
    s2.copy(s1)
    for _ in range(200):
        s1.step_pd(pin)
        s2.step_pd(pin)
    assert np.array_equal(s1.qpos(), s2.qpos())
    # hold with rows, with a write of 0 into the slide slots through the device pointer, and without rows
    L.cassie_batch_device_ptr.restype = C.c_void_p
    L.cassie_batch_device_ptr.argtypes = [C.c_void_p, C.c_char_p]
    ptr = L.cassie_batch_device_ptr(L.cassie_sim_batch(s2.c), b'mechanics')

    class _A:
        pass
    a = _A()
    a.__cuda_array_interface__ = dict(shape=(1, 192), typestr='<f8', data=(ptr, False), version=2)
    w = torch.as_tensor(a, device='cuda')
    w[0, MC_STIFF:MC_STIFF + 3] = 0.0
    torch.cuda.synchronize()
    drift = []
    for s in (s1, s2, s0):
        s.hold()
        q0 = s.qpos()[:3].copy()
        zero = P.pd_in_t()
        for _ in range(400):
            s.step_pd(zero)
        drift.append(float(np.abs(s.qpos()[:3] - q0).max()))
        s.release()
    print('pelvis drift under hold: with rows %.2e, with zeroed slide slots %.2e, without rows %.2e' % tuple(drift))
    assert max(drift) < 10 * drift[2] + 1e-6 and max(drift) < 1e-2, drift


def test_mixed_rows_follow_the_oracle(P, oracle_mod):
    """body-offset, actuator and mechanics rows in one fp64 batch, each environment against an oracle given all three: qpos within 1e-9 over 400
    saturating ticks"""
    from actuator_support import ActOracle
    O, n, model = oracle_mod, 3, 'cassie'
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    vals = batch_values(model, n, 80, base(b))
    bp = b.env_body_pos()
    names = table(model)['names_body']
    bp[1:, names.index('left-hip-pitch')] += [0.003, -0.002, 0.001]
    cr, rpm, dl = b.env_actuators()
    cr[2, :, 1] *= 0.7
    dl[1] = 3
    b.set_env_body_pos(bp)
    b.set_env_actuators(cr, rpm, dl)
    b.set_env_mechanics(*vals)
    os_ = []
    t = table(model)
    for e in range(n):   # the delay through ActOracle's delay line; ctrlrange, rpm, offsets and mechanics through the oracle's table
        o = ActOracle(O, model, cr[e], rpm[e], dl[e])
        o.o.close()
        user = t['actuator_user'].copy()
        user[:NU] = rpm[e]
        ctr = t['actuator_ctrlrange'].copy()
        ctr[:2 * NU] = cr[e].ravel()
        o.o = oracle_with(O, model, *[v[e] for v in vals], body_pos=bp[e], actuator_ctrlrange=ctr, actuator_user=user)
        o.line = np.ctypeslib.as_array(o.o.L.osim_torque_delay(o.o.h), shape=(NU, 6))
        os_.append(o)
    worst = 0.0
    for k in range(400):
        u = saturating_pd(O, k)
        b.set_pd(np.tile(np.concatenate([pd_row(u), np.zeros(P.PD_WIDTH - 50)]), (n, 1)))
        b.step(1)
        q = b.qpos()
        for e, o in enumerate(os_):
            o.step_pd(u)
            worst = max(worst, np.abs(q[e, :o.o.nq] - o.o.arr('qpos')).max())
    print('offsets + actuators + mechanics: worst qpos %.2e' % worst)
    assert worst <= 1e-9
    for o in os_:
        o.close()
    b.close()
