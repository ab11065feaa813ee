"""GPU: frame rows (cassie_batch_set_frames) -- the F_FR kernel instances against one oracle per sampled environment, bitwise neutrality of the frame
stages for every other output, snapshots, the zero-copy view and the verb's errors.  CPU twins (host emulation): tests/test_frames.py."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_env_geoms import placed_oracle
import ctypes as C

from test_frames import CFRC, VEL, all_frames, omodel, oracle_frames, oracle_jacobian

pytestmark = pytest.mark.gpu

MODELS = os.path.join(os.path.dirname(GOLDEN), '..', 'cassie-mujoco-sim_b200', 'models')


def _rows(P, n, on):
    return P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN) if on else P.pd_rows(n)


def _jitter(n, nq, seed=11):
    """per environment a pelvis placed up to 3 cm off and up to 2 cm higher than the reference pose"""
    rng = np.random.default_rng(seed)
    d = np.zeros((n, nq))
    d[:, 0:2] = rng.uniform(-0.03, 0.03, (n, 2))
    d[:, 2] = rng.uniform(0, 0.02, n)
    if nq > 35:   # cassie_tray_box.xml: the cup moves with the tray
        d[:, 35:38] = d[:, 0:3]
    return d


def _run_against_oracles(O, model, fp64, n=64, nsample=32, ticks=400, every=25, stairs=False, fall=True):
    P = product()
    b = P.CassieBatch(n, modelfile=os.path.join(MODELS, model + '.cmodel'), precision=P.FP64 if fp64 else P.FP32)
    names, kinds = all_frames(model)
    b.set_frames(names, kinds)
    q = b.qpos() + _jitter(n, b.qpos().shape[1])
    b.set_qpos(q)
    placements = [('box1', [0.05, 0.135, 0.04 - 0.1], None, [0.25, 0.1, 0.1])] if stairs else []
    for name, pos, quat, size in placements:
        b.set_env_geom_pose(name, pos=pos, quat=quat, size=size, mask=(np.arange(n) % 2 == 0).astype(np.uint8))
    b.set_pd(_rows(P, n, True))
    b.forward()
    sample = np.random.default_rng(5).choice(n, nsample, replace=False)
    m = omodel(model)
    oracles = []
    for e in sample:
        o = placed_oracle(O, placements) if (stairs and e % 2 == 0) else O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
        o.arr('qpos')[:] = q[e, :o.nq]
        o.forward()
        oracles.append(o)
    stance, motors_off = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    worst, scale, iters_ok = dict(pos=[], vel=[], cfrc=[]), dict(vel=0.0, cfrc=0.0), True
    for k in range(ticks):
        if fall and k == ticks // 2:
            b.set_pd(_rows(P, n, False))
        b.step(1)
        for o in oracles:
            o.step_pd(stance if (k < ticks // 2 or not fall) else motors_off)
        if fp64:
            it = b.counters()[sample, 3]
            iters_ok = iters_ok and all(int(it[i]) == o.get_int('solver_iter') for i, o in enumerate(oracles))
        if k % every == every - 1:
            fr = b.frames()
            for i, (e, o) in enumerate(zip(sample, oracles)):
                want = oracle_frames(o, m, names, kinds)
                worst['pos'].append(np.abs(fr[e, :, :VEL] - want[:, :VEL]).max())
                worst['vel'].append(np.abs(fr[e, :, VEL:CFRC] - want[:, VEL:CFRC]).max())
                worst['cfrc'].append(np.abs(fr[e, :, CFRC:] - want[:, CFRC:]).max())
                scale['vel'] = max(scale['vel'], np.abs(want[:, VEL:CFRC]).max())
                scale['cfrc'] = max(scale['cfrc'], np.abs(want[:, CFRC:]).max())
    assert int(b.counters()[:, 4].sum()) == 0   # no dropped contacts
    return {k: np.array(v) for k, v in worst.items()}, scale, iters_ok


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_fp64_frames_follow_the_oracle(oracle_mod, model):
    worst, scale, iters_ok = _run_against_oracles(oracle_mod, model, True)
    print(model, {k: v.max() for k, v in worst.items()}, scale)
    assert iters_ok
    assert worst['pos'].max() <= 1e-10 and worst['vel'].max() <= 1e-8 and worst['cfrc'].max() <= 1e-8


def test_fp64_frames_with_per_env_stairs(oracle_mod):
    worst, scale, iters_ok = _run_against_oracles(oracle_mod, 'cassie', True, stairs=True)
    print({k: v.max() for k, v in worst.items()}, scale)
    assert iters_ok
    assert worst['pos'].max() <= 1e-10 and worst['vel'].max() <= 1e-8 and worst['cfrc'].max() <= 1e-8


def test_fp32_frames_follow_the_oracle(oracle_mod):
    """fp32 on bench.py's config-2 controller (stance, fixed motor-PD targets): the single-precision trajectory itself drifts from the oracle, so
    the bars are on the poses (DESIGN.md section 3 style), with the velocities and forces within 1 % of their largest magnitude"""
    worst, scale, _ = _run_against_oracles(oracle_mod, 'cassie', False, n=256, nsample=64, ticks=600, fall=False)
    print({k: (np.median(v), v.max()) for k, v in worst.items()}, scale)
    assert np.median(worst['pos']) <= 1e-5 and worst['pos'].max() <= 1e-3
    assert worst['vel'].max() <= 1e-2 * scale['vel'] and worst['cfrc'].max() <= 1e-2 * scale['cfrc']


@pytest.mark.parametrize('fp64', [True, False])
def test_frames_change_no_other_output(fp64):
    """the F_FR instance against the shipped extended instance: qpos, qvel, obs, aux and the counters bitwise equal over 1000 ticks"""
    P = product()
    n = 128
    a, b = (P.CassieBatch(n, precision=P.FP64 if fp64 else P.FP32) for _ in range(2))
    names, kinds = all_frames('cassie')
    b.set_frames(names, kinds)
    for x in (a, b):
        x.enable_aux(True)
        x.set_qpos(x.qpos() + _jitter(n, x.qpos().shape[1]))
        x.set_pd(_rows(P, n, True))
        x.forward()
    for k in range(1000):
        if k == 500:
            for x in (a, b):
                x.set_pd(_rows(P, n, False))
        a.step(1)
        b.step(1)
        if k % 50 == 49:
            for f in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
                assert np.array_equal(getattr(a, f)(), getattr(b, f)()), (k, f)
    assert np.abs(b.frames()[:, :, CFRC:]).max() > 0


def test_feet_frames_equal_aux_and_multi_tick_launches():
    """foot frames bitwise aux's foot velocities / forces of the same launch, also after multi-tick launches"""
    P = product()
    b = P.CassieBatch(64, precision=P.FP64)
    b.enable_aux(True)
    b.set_frames(['left-foot', 'right-foot'])
    b.set_pd(_rows(P, 64, True))
    b.forward()
    for _ in range(20):
        b.step(10)
        fr, aux = b.frames(), b.aux()
        assert np.array_equal(fr[:, 0, VEL:CFRC], aux[:, 30:36]) and np.array_equal(fr[:, 1, VEL:CFRC], aux[:, 36:42])
        assert np.array_equal(fr[:, 0, CFRC:CFRC + 6], aux[:, 0:6]) and np.array_equal(fr[:, 1, CFRC:CFRC + 6], aux[:, 6:12])


def test_snapshot_restores_frames_and_torch_view():
    import torch
    P = product()
    n = 32
    b = P.CassieBatch(n, precision=P.FP32)
    names, kinds = all_frames('cassie')
    b.set_frames(names, kinds)
    b.set_pd(_rows(P, n, True))
    b.forward()
    b.step(50)
    snap = b.get_state()
    before = b.frames()
    b.step(50)
    assert not np.array_equal(before, b.frames())
    b.set_state(snap)
    assert np.array_equal(before, b.frames())
    b.step(3)
    b.sync()
    v = b.torch_view('frames')
    assert tuple(v.shape) == (n, len(names) * 20) and v.dtype == torch.float32
    assert np.array_equal(v.cpu().numpy().reshape(n, len(names), 20).astype(np.float64), b.frames())
    b.free_state(snap)


def test_set_frames_errors_and_clear():
    P = product()
    b = P.CassieBatch(4, precision=P.FP32)
    for names, kinds in ((['no-such-body'], [0]), (['left-toe'], [0]), (['cassie-pelvis'], [2]), (['cassie-pelvis'] * 65, [0] * 65)):
        with pytest.raises(RuntimeError):
            b.set_frames(names, kinds)
        assert b.nframes() == 0
    b.set_frames(['world', 'cassie-pelvis', 'left-toe'], [0, 0, 1])
    assert b.nframes() == 3 and b.row_width('frames') == 60
    with pytest.raises(RuntimeError):
        b.set_frames(['cassie-pelvis', 'nope'])
    assert b.nframes() == 3   # a refused call changes nothing
    b.step(2)
    fr = b.frames()
    assert np.array_equal(fr[:, 0, :7], np.tile([0, 0, 0, 1, 0, 0, 0], (4, 1)))   # the world frame
    b.set_frames([])
    assert b.nframes() == 0
    with pytest.raises(RuntimeError):
        b.frames()
    b.step(2)


def test_frame_jacobian_tray_box(oracle_mod):
    """mode 4 on cassie_tray_box (38 columns): every body and the site against the oracle at the batch's current states, and no state written"""
    P = product()
    n, model = 16, 'cassie_tray_box'
    b = P.CassieBatch(n, modelfile=os.path.join(MODELS, model + '.cmodel'), precision=P.FP64)
    names, kinds = all_frames(model)
    b.set_frames(names, kinds)
    b.set_qpos(b.qpos() + _jitter(n, b.qpos().shape[1]))
    b.set_pd(_rows(P, n, True))
    b.forward()
    b.step(150)
    before = [b.qpos(), b.qvel(), b.obs(), b.frames(), b.counters()]
    worst = 0.0
    for f, (name, kind) in enumerate(zip(names, kinds)):
        jp, jr = b.frame_jacobian(f)
        assert jp.shape == (n, 3, 38)
        for e in (0, 5, 11):
            wp, wr = oracle_jacobian(oracle_mod, model, b.qpos()[e], name, kind)
            worst = max(worst, np.abs(jp[e] - wp).max(), np.abs(jr[e] - wr).max())
    print(worst)
    assert worst <= 1e-10
    for x, y in zip(before, [b.qpos(), b.qvel(), b.obs(), b.frames(), b.counters()]):
        assert np.array_equal(x, y)
    v = b.torch_view('frame_jac')
    assert tuple(v.shape) == (n, 240)
    with pytest.raises(RuntimeError):
        b.frame_jacobian(len(names))


def _y_bytes(y):
    return bytes(memoryview(y).cast('B'))


def test_legacy_sim_is_bitwise_a_frameless_batch_of_one():
    """a cassie_sim_t (fp64, every body and site tracked: the F_FR instance) against a batch of one without frames on the shipped extended instance:
    qpos, qvel, state_out_t and the aux row bitwise equal over 1000 ticks"""
    P = product()
    c = P.CassieSim()
    b = P.CassieBatch(1, precision=P.FP64)
    b.enable_aux(True)
    b.forward()
    b.enable_estimator_device(True)
    pu = _pd_in(P)
    arr = (P.pd_in_t * 1)(pu)
    for k in range(1000):
        y = c.step_pd(pu)
        yb = b.step_pd(arr)
        if k % 50 == 49:
            assert np.array_equal(c.qpos(), b.qpos()[0]) and np.array_equal(c.qvel(), b.qvel()[0]), k
            assert _y_bytes(y) == _y_bytes(yb[0]), k
            assert np.array_equal(c.foot_forces_raw(), b.aux()[0, 0:12]), k


def _pd_in(P):
    pu = P.pd_in_t()
    for side, leg in enumerate((pu.leftLeg, pu.rightLeg)):
        for i in range(5):
            leg.motorPd.pTarget[i] = PD_TARGET[5 * side + i]
            leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_PGAIN[i], PD_DGAIN[i]
    return pu


def test_legacy_frame_verbs_follow_the_oracle(oracle_mod):
    """cassie_sim_xpos / xquat (pointer arithmetic across bodies, as &d->xpos[3 * id]), site_xpos / site_xquat, body_velocities, body_contact_force,
    the three Jacobian verbs and relative_pose against the oracle; a snapshot restore brings the frame mirrors back"""
    P, O = product(), oracle_mod
    m = omodel('cassie')
    names, kinds = all_frames('cassie')
    nb = len(m['names_body'])
    c, o = P.CassieSim(), O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    pu, u = _pd_in(P), O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    L = c.L
    L.cassie_sim_xpos.restype = L.cassie_sim_xquat.restype = C.POINTER(C.c_double)
    L.cassie_sim_xpos.argtypes = L.cassie_sim_xquat.argtypes = [C.c_void_p, C.c_char_p]
    worst = dict(pos=0.0, vel=0.0, cfrc=0.0, jac=0.0)
    for k in range(300):
        c.step_pd(pu)
        o.step_pd(u)
        if k % 50 == 49:
            want = oracle_frames(o, m, names, kinds)
            px, pq = L.cassie_sim_xpos(c.c, b'world'), L.cassie_sim_xquat(c.c, b'world')
            for bi in range(nb):
                worst['pos'] = max(worst['pos'], max(abs(px[3 * bi + j] - want[bi, j]) for j in range(3)), max(abs(pq[4 * bi + j] - want[bi, 3 + j]) for j in range(4)))
                v, f = np.zeros(6), np.zeros(6)
                c.body_vel(v, names[bi])
                c.get_body_contact_force(f, names[bi])
                worst['vel'] = max(worst['vel'], np.abs(v - want[bi, VEL:CFRC]).max())
                worst['cfrc'] = max(worst['cfrc'], np.abs(f - want[bi, CFRC:CFRC + 6]).max())
            for si, name in enumerate(m['names_site']):
                worst['pos'] = max(worst['pos'], np.abs(c.get_site_xpos(name) - want[nb + si, :3]).max(), np.abs(np.array(c.get_site_quat(name)) - want[nb + si, 3:7]).max())
            q = c.qpos()
            for name, kind in (('cassie-pelvis', 0), ('left-foot', 0), ('right-toe', 1)):
                wp, wr = oracle_jacobian(O, 'cassie', q, name, kind)
                if kind == 0:
                    jp, jr = c.get_jacobian_full(name)
                    worst['jac'] = max(worst['jac'], np.abs(c.get_jacobian(name) - wp.ravel()).max())
                else:
                    jp, jr = c.get_jacobian_full_site(name)
                worst['jac'] = max(worst['jac'], np.abs(jp - wp.ravel()).max(), np.abs(jr - wr.ravel()).max())
    print(worst)
    assert worst['pos'] <= 1e-10 and worst['vel'] <= 1e-8 and worst['cfrc'] <= 1e-8 and worst['jac'] <= 1e-10
    # relative pose: pose 2 in the frame of pose 1
    p1, p2 = np.r_[c.xpos('cassie-pelvis'), c.xquat('cassie-pelvis')], np.r_[c.xpos('left-foot'), c.xquat('left-foot')]
    rel = np.zeros(7)
    c.get_object_relative_pose(p1, p2, rel)
    w, x, y, z = p1[3:]
    R = np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                  [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])
    assert np.abs(rel[:3] - R.T @ (p2[:3] - p1[:3])).max() < 1e-12
    # snapshot restore: the frame mirrors describe the restored state
    s = c.get_state()
    keep = [c.xpos(nm) for nm in m['names_body']]
    for _ in range(40):
        c.step_pd(pu)
    assert not np.array_equal(keep[1], c.xpos('cassie-pelvis'))
    c.set_state(s)
    assert all(np.array_equal(a, c.xpos(nm)) for a, nm in zip(keep, m['names_body']))
    with pytest.raises(KeyError):
        c.xpos('no-such-body')
    assert not c.get_jacobian('no-such-body').any()
