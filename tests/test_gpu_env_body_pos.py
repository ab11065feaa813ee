"""GPU: per-environment body offsets (cassie_batch_set_env_body_pos, the F_BP instances) and the legacy body-position verbs, against the fp64 oracle
with the same body_pos (a temporary copy of its model table, tests/test_env_body_pos.py) and against the host emulation of the same source."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
import raycast_support as RS
from test_accelerations import oracle_row, split
from test_dynamics import full_m
from test_env_body_pos import BodyRowSim, _dp, offsets, oracle_with, table
from test_frames import CFRC, VEL, all_frames, omodel, oracle_frames
from test_gpu_raycast import slot_scene

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def P():
    return product()


def batch_offsets(model, n, seed):
    """[n, nbody, 3]: environment e gets offsets(model, seed + e); environment 0 the model's"""
    _, _, bp, _ = table(model)
    return np.stack([bp] + [offsets(model, seed + e) for e in range(1, n)])


def test_four_envs_fp64_with_set_const(P, oracle_mod):
    """4 environments, each its own offsets, one also its own masses == 4 oracle sims with the same body_pos (and masses); a masked set_const with
    state reset on two of them, then 250 more ticks"""
    O, n, model = oracle_mod, 4, 'cassie'
    pos = batch_offsets(model, n, 40)
    os_ = [oracle_with(O, model, pos[e]) for e in range(n)]
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    b.set_env_body_pos(pos)
    assert np.array_equal(b.env_body_pos(), pos)
    mass = b.get_model('body_mass')
    mass[2] *= 1.1
    b.set_model('body_mass', mass)
    os_[2].model_arr('body_mass')[:] = mass[2]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    for o in os_:
        o.forward()
    b.reset()
    for _ in range(250):
        for o in os_:
            o.step_pd(u)
    b.step(250)
    q = b.qpos()
    for i, o in enumerate(os_):
        assert np.abs(q[i] - o.arr('qpos')).max() < 1e-9, i
    mask = np.array([0, 1, 0, 1], dtype=np.uint8)
    before = b.qpos()
    b.set_const(mask, reset_state=True)
    assert np.array_equal(b.qpos()[[0, 2]], before[[0, 2]])
    for i in (1, 3):
        os_[i].set_const()
    for _ in range(250):
        for o in os_:
            o.step_pd(u)
    b.step(250)
    q = b.qpos()
    for i, o in enumerate(os_):
        assert np.abs(q[i] - o.arr('qpos')).max() < 1e-9, i
    b.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_mass'])
def test_fp32_4096_sampled_against_the_oracle(P, oracle_mod, model):
    """4096 fp32 environments with seeded offsets; 64 sampled environments replayed in the oracle for 600 ticks.  Bars over the sample's worst qpos
    error: median <= 1e-5, p90 <= 1e-4, worst <= 1e-3; no contact dropped"""
    n, T = 4096, 600
    _, _, bp, _ = table(model)
    rng = np.random.default_rng(77)
    names = table(model)[0]
    pos = np.broadcast_to(bp, (n, len(names), 3)).copy()
    movable = [names.index(x) for x in (('left-hip-roll', 'right-hip-roll', 'left-hip-pitch', 'right-hip-pitch') if model == 'cassie' else ('load_mass',))]
    scale = 0.005 if model == 'cassie' else 0.02
    for b_ in movable:
        pos[:, b_] += rng.uniform(-scale, scale, (n, 3))
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32)
    b.set_env_body_pos(pos)
    b.reset()
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.step(T)
    q = b.qpos()
    assert (b.counters()[:, 4] == 0).all()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    errs = []
    for e in np.random.default_rng(5).choice(n, 64, replace=False):
        o = oracle_with(oracle_mod, model, pos[e])
        o.forward()
        for _ in range(T):
            o.step_pd(u)
        errs.append(np.abs(q[e] - o.arr('qpos')).max())
        o.close()
    errs = np.array(errs)
    print(model, 'median %.2e p90 %.2e worst %.2e' % (np.median(errs), np.percentile(errs, 90), errs.max()))
    assert np.median(errs) <= 1e-5 and np.percentile(errs, 90) <= 1e-4 and errs.max() <= 1e-3
    b.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_launch_modes_follow_the_oracle(P, oracle_mod, fp32):
    """frames (every body), acceleration rows and dynamics rows with offsets (the F_BP | F_FR instances: d157, and f157 in fp32) against oracles with
    the same body_pos stepped alongside: fp64 frame poses within 1e-10, velocities and contact forces within 1e-8, qacc within 1e-8 of its largest
    magnitude, M within 1e-12 of its largest entry; fp32 frame poses within 1e-3 and M within 1e-5 (at the batch's own state)"""
    n, model, ticks = 3, 'cassie', 200
    pos = batch_offsets(model, n, 60)
    m = omodel(model)
    names, kinds = all_frames(model)
    nbn = len(m['names_body'])
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32 if fp32 else P.FP64)
    b.set_env_body_pos(pos)
    b.set_frames(names[:nbn], kinds[:nbn])
    b.enable_accelerations()
    b.reset()
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    os_ = [oracle_with(oracle_mod, model, pos[e]) for e in range(n)]
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
        d = oracle_with(oracle_mod, model, pos[e])   # M at the batch's own state
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
    assert np.abs(fr[1, :, :3] - fr[0, :, :3]).max() > 1e-3   # the offsets moved the bodies
    for o in os_:
        o.close()
    b.close()


BOX = 1   # cassie.xml's box1, in the reference's geom numbering


@pytest.mark.parametrize('fp32', [False, True])
def test_broad_phase_covers_a_lengthened_leg(P, oracle_mod, fp32):
    """the left tarsus three times its length, the robot lifted 0.7 m, and a box placed per environment (F_EG | F_BP: d15f / f15f) around the left foot,
    farther from the pelvis than the model's robot bound plus the box's bounding radius: the broad phase would cull it with the model's bound.  The
    kernel must find the oracle's contacts; a rebuild of the block (cassie_batch_set_timestep) must keep the recomputed bound"""
    names, nb, bp, _ = table('cassie')
    n, hs = 2, 0.05
    long_ = bp.copy()
    long_[names.index('left-tarsus')] *= 3.0
    pos = np.stack([bp, long_])
    q0 = None
    boxes = []
    for e in range(n):   # the box around each environment's left foot (the oracle's kinematics at the lifted initial pose)
        o = oracle_with(oracle_mod, 'cassie', pos[e])
        o.arr('qpos')[2] += 0.7
        o.forward()
        q0 = o.arr('qpos').copy() if q0 is None else q0
        xp = o.arr('xpos').reshape(-1, 3)
        boxes.append((xp[names.index('left-foot')].copy(), xp[1].copy()))
        o.close()
    s = BodyRowSim('cassie')
    reach = np.zeros(2)
    s.L.emu_bp_reach(s.h, _dp(bp), reach.ctypes.data_as(C.POINTER(C.c_double)))
    s.close()
    foot, pelvis = boxes[1]
    assert np.linalg.norm(foot - pelvis) - np.sqrt(3) * hs > reach[0] + 0.02   # culled by the model's bound
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32 if fp32 else P.FP64)
    b.set_env_body_pos(pos)
    b.set_env_geom_pose('box%d' % BOX, pos=np.stack([c for c, _ in boxes]), size=[hs, hs, hs])
    want = []
    for e in range(n):
        o = oracle_with(oracle_mod, 'cassie', pos[e], rbound={BOX: np.sqrt(3) * hs})
        o.model_arr('geom_pos').reshape(-1, 3)[BOX] = boxes[e][0]
        o.model_arr('geom_size').reshape(-1, 3)[BOX] = hs
        o.arr('qpos')[:] = q0
        o.forward()
        assert sum(1 for c in o.contacts() if BOX in (c['geom1'], c['geom2'])) > 0, e   # the foot is in the box
        want.append(o.get_int('ncon'))
        o.close()
    qb = np.broadcast_to(q0, (n, len(q0))).copy()
    for rebuilt in (False, True):   # the bound the setter wrote, then the bound a rebuild of the block keeps
        if rebuilt:
            b.set_timestep(float(omodel('cassie')['opt_timestep'][0]))
        b.set_qpos(qb)
        b.forward()
        got = [int(x) for x in b.counters()[:, 1]]
        assert got == want, (rebuilt, got, want)
    b.close()


def test_env_terrain_with_offsets_follows_the_oracle(P, oracle_mod):
    """per-environment terrain rows (the shared placement, entry 0 of a flat bank) with offsets: the F_ALL | F_EG | F_TR | F_BP instance d17f against
    oracles of cassie_hfield.xml with the same body_pos, 200 ticks within 1e-9"""
    model, n = 'cassie_hfield', 2
    names, nb, bp, _ = table(model)
    pos = np.stack([bp, bp])
    pos[1, names.index('left-hip-roll')] += [0.004, -0.003, 0.002]
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    b.set_env_body_pos(pos)
    b.set_env_hfield(terrain=0)
    b.reset()
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.step(200)
    q = b.qpos()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for e in range(n):
        o = oracle_with(oracle_mod, model, pos[e])
        o.forward()
        for _ in range(200):
            o.step_pd(u)
        assert np.abs(q[e] - o.arr('qpos')).max() < 1e-9, e
        o.close()
    assert np.abs(q[1] - q[0]).max() > 1e-5
    b.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_model_rows_and_clear(P, fp32):
    """rows at the model's values follow no rows (separately compiled instances: 1e-11 fp64, 1e-5 fp32); set-then-clear is bitwise never-set"""
    prec, tol = (P.FP32, 1e-5) if fp32 else (P.FP64, 1e-11)
    _, _, bp, _ = table('cassie')
    a, b, c = (P.CassieBatch(64, precision=prec) for _ in range(3))
    b.set_env_body_pos(bp)
    c.set_env_body_pos(batch_offsets('cassie', 64, 3))
    c.clear_env_body_pos()
    assert np.array_equal(c.env_body_pos(), b.env_body_pos())
    for x in (a, b, c):
        x.set_pd(P.pd_rows(64, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        x.step(300)
    assert np.abs(a.qpos() - b.qpos()).max() < tol
    assert np.array_equal(a.qpos(), c.qpos()) and np.array_equal(a.obs(), c.obs())
    for x in (a, b, c):
        x.close()


def test_aos_entry_point_equals_compact_path(P):
    """cassie_sim_step_pd_batch with offsets == the compact path with the same offsets and inputs, bit for bit"""
    n = 4096
    pos = np.broadcast_to(table('cassie')[2], (n, 26, 3)).copy()
    pos[:, 2] += np.random.default_rng(8).uniform(-0.005, 0.005, (n, 3))
    a, b = P.CassieBatch(n, precision=P.FP32), P.CassieBatch(n, precision=P.FP32)
    for x in (a, b):
        x.set_env_body_pos(pos)
    b.enable_estimator_device(True)
    pd = (P.pd_in_t * n)()
    for e in range(n):
        for side, leg in enumerate((pd[e].leftLeg, pd[e].rightLeg)):
            for i in range(5):
                leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    for k in range(200):
        a.step_pd(pd)
        b.step(1)
    assert np.array_equal(a.qpos(), b.qpos()) and np.array_equal(a.obs(), b.obs())
    a.close()
    b.close()


def test_refusals_reset_and_snapshots(P):
    """refused inputs change nothing; reset and snapshot restore keep the rows"""
    model = 'cassie_tray_box'
    names, nb, bp, weld = table(model)
    b = P.CassieBatch(4, modelfile=P.model_path(model), precision=P.FP64)
    good = batch_offsets(model, 4, 20)
    b.set_env_body_pos(good)
    for body in (0, nb - 1, [x for x in range(1, nb) if weld[x] == 0][0] if (weld[1:] == 0).any() else 0):
        bad = good.copy()
        bad[2, body, 0] += 0.01
        with pytest.raises(RuntimeError):
            b.set_env_body_pos(bad)
        assert np.array_equal(b.env_body_pos(), good)
    bad = good.copy()
    bad[1, 3, 2] = np.nan
    with pytest.raises(RuntimeError):
        b.set_env_body_pos(bad)
    assert np.array_equal(b.env_body_pos(), good)
    b.step(50)
    s = b.get_state()
    b.reset()
    assert np.array_equal(b.env_body_pos(), good)
    b.set_state(s)
    assert np.array_equal(b.env_body_pos(), good)
    b.close()


def test_rays_and_depth_follow_the_emulation(P, oracle_mod):
    """height scans and depth images with a per-environment pelvis offset: the F_BP rows on the device against the host emulation of the same row, and
    the height scans against the ray oracle cast from the oracle's root pose with the same body_pos"""
    scene = slot_scene('cassie')
    n = 4
    names, nb, bp, _ = table('cassie')
    pos = np.broadcast_to(bp, (n, nb, 3)).copy()
    pos[:, 1] += np.array([[0, 0, 0], [0.03, -0.02, 0.05], [-0.04, 0.01, 0.02], [0.0, 0.05, -0.03]])
    b = P.CassieBatch(n, precision=P.FP64)
    b.set_env_body_pos(pos)
    b.reset()
    k = 24
    ang = np.linspace(0, 2 * np.pi, k, endpoint=False)
    org = np.stack([0.3 * np.cos(ang), 0.3 * np.sin(ang), np.zeros(k)], 1)
    b.set_rays(org, np.tile([0.0, 0.0, -1.0], (k, 1)), frame='root', max_dist=3.0)
    b.raycast()
    rays = b.rays()
    b.set_camera(body='cassie-pelvis', pos=[0.1, 0, 0.1], quat=[0.5, -0.5, 0.5, -0.5], fovy=70.0, width=24, height=16, zfar=5.0)
    b.render_depth()
    depth = b.depth()
    q = b.qpos()
    for e in range(n):
        s = BodyRowSim('cassie')
        s.set_env_body_pos(pos[e])
        s.L.emu_set.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.c_int]
        qq = np.zeros(64)
        qq[:35] = q[e]
        s.L.emu_set(s.h, b'qpos', qq.ctypes.data_as(C.POINTER(C.c_double)), 64)
        s.forward()
        out = np.zeros(k * 4)
        frame = np.ones(k, dtype=np.int32)
        s.L.emu_bp_rays(s.h, frame.ctypes.data_as(C.POINTER(C.c_int)), org.ctypes.data_as(C.POINTER(C.c_double)),
                        np.ascontiguousarray(np.tile([0.0, 0.0, -1.0], (k, 1))).ctypes.data_as(C.POINTER(C.c_double)),
                        np.full(k, 3.0).ctypes.data_as(C.POINTER(C.c_double)), k, out.ctypes.data_as(C.POINTER(C.c_double)))
        assert np.abs(out.reshape(k, 4) - rays[e]).max() < 1e-11, e
        img = np.zeros(24 * 16)
        s.L.emu_bp_camera(s.h, names.index('cassie-pelvis'), np.array([0.1, 0, 0.1]).ctypes.data_as(C.POINTER(C.c_double)),
                          np.array([0.5, -0.5, 0.5, -0.5]).ctypes.data_as(C.POINTER(C.c_double)), 70.0, 24, 16, 5.0, img.ctypes.data_as(C.POINTER(C.c_double)))
        assert np.abs(img.reshape(16, 24) - depth[e]).max() < 1e-11, e
        s.close()
        o = oracle_with(oracle_mod, 'cassie', pos[e])   # the ray oracle, from the oracle's root pose with the same body_pos
        o.arr('qpos')[:] = q[e, :o.nq]
        o.forward()
        rp, R = RS.root_pose(o, names.index('cassie-pelvis'))
        o.close()
        ow, dw = RS.world_rays(RS.ROOT, org, np.tile([0.0, 0.0, -1.0], (k, 1)), rp, R)
        ref = RS.oracle_cast(scene, ow, dw, 3.0)
        assert np.abs(rays[e][:, :2] - ref[:, :2]).max() < 1e-11 and (ref[:, 0] > 0).all(), e
    assert np.abs(rays[1] - rays[0]).max() > 1e-3
    b.close()


def sim_pd(P):
    """the standing PD input of the legacy object"""
    u = P.pd_in_t()
    for side, leg in enumerate((u.leftLeg, u.rightLeg)):
        for i in range(5):
            leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
    return u


def test_legacy_verbs(P, oracle_mod):
    """writes through the borrowed pointer and set_body_pos, then set_const, then 400 ticks == the oracle with that body_pos and mj_setConst;
    an unknown name raises; moving the floor of cassie_hfield.xml moves the contacts the robot stands on as in the oracle"""
    names, nb, bp, _ = table('cassie')
    p = bp.copy()
    p[names.index('left-hip-roll')] += [0.004, -0.003, 0.002]
    p[names.index('right-hip-pitch')] += [-0.003, 0.0, 0.004]
    s = P.CassieSim(P.model_path('cassie'))
    ptr = s.L.cassie_sim_get_body_name_pos(s.c, b'left-hip-roll')
    for c in range(3):
        ptr[c] = p[names.index('left-hip-roll')][c]
    s.set_body_pos('right-hip-pitch', p[names.index('right-hip-pitch')])
    assert np.array_equal(s.get_body_pos('right-hip-pitch'), p[names.index('right-hip-pitch')])
    s.set_const()
    o = oracle_with(oracle_mod, 'cassie', p)
    o.set_const()
    u, us = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), sim_pd(P)
    for _ in range(400):
        s.step_pd(us)
        o.step_pd(u)
    assert np.abs(s.qpos() - o.arr('qpos')).max() < 1e-9
    with pytest.raises(RuntimeError):
        s.get_body_pos('no-such-body')
    # the floor of cassie_hfield.xml (the static body carrying the height field) moved 3 cm down: the robot lands lower, as in the oracle
    hn, _, hbp, _ = table('cassie_hfield')
    f = hn.index('floor')
    hp = hbp.copy()
    hp[f, 2] -= 0.03
    h = P.CassieSim(P.model_path('cassie_hfield'))
    h.set_body_pos('floor', hp[f])
    oh, o0 = oracle_with(oracle_mod, 'cassie_hfield', hp), oracle_mod.OracleSim(os.path.join(GOLDEN, 'cassie_hfield.omodel'))
    for x in (oh, o0):
        x.forward()
    for _ in range(500):   # the drop onto the height field: contacts from about tick 400 on
        h.step_pd(us)
        oh.step_pd(u)
        o0.step_pd(u)
    assert np.abs(h.qpos() - oh.arr('qpos')).max() < 1e-9
    assert oh.get_int('ncon') > 0 and o0.arr('qpos')[2] - h.qpos()[2] > 5e-3, (h.qpos()[2], o0.arr('qpos')[2])   # it landed lower than on the unmoved floor
    oh.close()
    o0.close()
    o.close()
    del h, s   # CassieSim frees its simulator when collected (cassie_sim_free)
