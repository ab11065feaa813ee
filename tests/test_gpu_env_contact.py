"""GPU: per-environment contact softness (cassie_batch_set_env_contact, the F_CT instances: solref, solimp and solmix per collision geom), against the
fp64 oracle given the same geom_solref, geom_solimp and geom_solmix (a temporary copy of its model table, tests/contact_support.py)."""
import ctypes as C

import numpy as np
import pytest

from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product
from contact_support import colliding, contact_oracle, random_contact
from mechanics_support import table
from test_accelerations import oracle_row, split
from test_frames import CFRC, VEL, all_frames, omodel, oracle_frames

pytestmark = pytest.mark.gpu
PARTS = ('solref', 'solimp', 'solmix')
CT_SLOT, CT_SOLREF = 8, 0


@pytest.fixture(scope='module')
def P():
    return product()


def base(b):
    """the model's values as the batch reports them without rows (solref, solimp, solmix)"""
    m = b.env_contact()
    return [m[k][0] for k in PARTS]


def batch_values(model, n, seed, b0):
    """[n, ...] per part: environment e gets random_contact(model, seed + e) from the batch's model values; environment 0 the model's"""
    vals = [b0] + [random_contact(model, seed + e, b0) for e in range(1, n)]
    return [np.stack([v[p] for v in vals]) for p in range(3)]


def _pd(P, b, n):
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))


def test_four_envs_fp64(P, oracle_mod):
    """4 environments, each its own contact rows, one also its own friction rows and one its own floor tilt (d13df) == 4 oracles with the same tables:
    qpos within 1e-9 and equal PGS iteration counts over 500 ticks"""
    O, n, model = oracle_mod, 4, 'cassie'
    t = table(model)
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    vals = batch_values(model, n, 40, base(b))
    b.set_env_contact(*vals)
    got = b.env_contact()
    assert all(np.array_equal(got[k], v) for k, v in zip(PARTS, vals))
    fr = b.get_model('geom_friction')
    fr[1, 0::3] *= 0.6
    b.set_model('geom_friction', fr)
    tilt = np.array([np.cos(0.01), np.sin(0.01), 0.0, 0.0])
    b.set_env_geom_pose('floor', quat=np.array([[1.0, 0, 0, 0], [1.0, 0, 0, 0], tilt, [1.0, 0, 0, 0]]))
    gq = t['geom_quat'].reshape(-1, 4).copy()
    gq[0] = tilt
    os_ = [contact_oracle(O, model, *[v[e] for v in vals], **({'geom_friction': fr[e]} if e == 1 else {'geom_quat': gq} if e == 2 else {})) for e in range(n)]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    _pd(P, b, n)
    for o in os_:
        o.forward()
    b.reset()
    same, worst = True, 0.0
    for _ in range(500):
        b.step(1)
        it = b.counters()[:, 3]
        q = b.qpos()
        for e, o in enumerate(os_):
            o.step_pd(u)
            same = same and int(it[e]) == o.get_int('solver_iter')
            worst = max(worst, float(np.abs(q[e, :o.nq] - o.arr('qpos')).max()))
    print('four fp64 environments: worst qpos %.2e' % worst)
    assert worst < 1e-9 and same, (worst, same)
    assert np.abs(b.qpos()[1] - b.qpos()[0]).max() > 1e-5
    for o in os_:
        o.close()
    b.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_mass'])
def test_fp32_4096_sampled_against_the_oracle(P, oracle_mod, model):
    """4096 fp32 environments with seeded contact rows (f13c4); 64 sampled environments replayed in the oracle for 600 ticks.  Bars over the sample's
    worst qpos error (DESIGN.md section 3): median <= 1e-5, p90 <= 3e-5, worst <= 1e-3; no contact dropped"""
    n, T = 4096, 600
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32)
    vals = batch_values(model, n, 1000, base(b))
    b.set_env_contact(*vals)
    b.reset()
    _pd(P, b, n)
    b.step(T)
    q = b.qpos()
    assert (b.counters()[:, 4] == 0).all()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    errs = []
    for e in np.random.default_rng(5).choice(n, 64, replace=False):
        o = contact_oracle(oracle_mod, model, *[v[e] for v in vals])
        o.forward()
        for _ in range(T):
            o.step_pd(u)
        errs.append(np.abs(q[e, :o.nq] - o.arr('qpos')).max())
        o.close()
    errs = np.array(errs)
    print(model, 'median %.2e p90 %.2e worst %.2e' % (np.median(errs), np.percentile(errs, 90), errs.max()))
    assert np.median(errs) <= 1e-5 and np.percentile(errs, 90) <= 3e-5 and errs.max() <= 1e-3
    b.close()


# (model, precision, what else the batch carries) -> the instance it runs: each of the seven F_CT instances, against its F_MC twin
ROUTES = [('cassie', 'fp32', None, 'f13c4'), ('cassie', 'fp32', 'frames', 'f13d7'), ('cassie', 'fp64', None, 'd13d7'), ('cassie', 'fp32', 'geom', 'f13df'),
          ('cassie', 'fp64', 'geom', 'd13df'), ('cassie_hfield', 'fp32', 'hfield', 'f13ff'), ('cassie_hfield', 'fp64', 'hfield', 'd13ff')]


@pytest.mark.parametrize('model,prec,extra,tag', ROUTES, ids=[r[3] for r in ROUTES])
def test_model_rows_are_bitwise_the_mechanics_twin(P, model, prec, extra, tag):
    """model-valued contact rows against the same batch with model-valued mechanics rows only (the F_MC twin) over 400 ticks: qpos, qvel, obs, aux and
    the counters bit for bit"""
    n = 64
    bs = [P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32 if prec == 'fp32' else P.FP64) for _ in range(2)]
    for x in bs:
        x.enable_aux()
        if extra == 'frames':
            x.set_frames(['left-foot', 'right-foot'])
        elif extra == 'geom':
            x.set_env_geom_pose('floor', pos=[0.0, 0.0, 0.0])
        elif extra == 'hfield':
            x.set_env_hfield(terrain=0)
    a, b = bs
    a.set_env_mechanics(*[a.env_mechanics()[k] for k in ('inertia', 'armature', 'stiffness', 'springref')])
    b.set_env_contact(*base(b))
    for x in bs:
        x.reset()
        _pd(P, x, n)
        x.step(400)
    for name in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
        assert np.array_equal(getattr(a, name)(), getattr(b, name)()), (tag, name)
    assert b.device_ptr('contact') and not a.device_ptr('contact')
    a.close()
    b.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_launch_modes_follow_the_oracle(P, oracle_mod, fp32):
    """frames (every body, with their contact forces), the aux foot / toe / heel forces, and acceleration rows with contact rows (d13d7, f13d7) against
    oracles with the same tables: fp64 frame poses within 1e-10, velocities and contact forces within 1e-8, foot forces within 1e-8, qacc within 1e-8 of
    its largest magnitude; fp32 frame poses within 1e-3"""
    n, model, ticks = 3, 'cassie', 300
    m = omodel(model)
    names, kinds = all_frames(model)
    nbn = len(m['names_body'])
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32 if fp32 else P.FP64)
    vals = batch_values(model, n, 60, base(b))
    b.set_env_contact(*vals)
    b.set_frames(names[:nbn], kinds[:nbn])
    b.enable_accelerations()
    b.enable_aux()
    b.reset()
    _pd(P, b, n)
    os_ = [contact_oracle(oracle_mod, model, *[v[e] for v in vals]) for e in range(n)]
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for o in os_:
        o.forward()
    for _ in range(ticks):
        b.step(1)
        for o in os_:
            o.step_pd(u)
    fr, qa, aux = b.frames(), b.qacc(), b.aux()
    for e, o in enumerate(os_):
        want = oracle_frames(o, m, names[:nbn], kinds[:nbn])
        dpos = np.abs(fr[e, :, :VEL] - want[:, :VEL]).max()
        if fp32:
            assert dpos <= 1e-3, (e, dpos)
            continue
        assert dpos <= 1e-10, (e, dpos)
        assert np.abs(fr[e, :, VEL:CFRC] - want[:, VEL:CFRC]).max() <= 1e-8 and np.abs(fr[e, :, CFRC:] - want[:, CFRC:]).max() <= 1e-8, e
        assert np.abs(want[:, CFRC:]).max() > 1.0   # the feet carry the robot
        toe, heel = o.heeltoe_forces()
        assert np.abs(aux[e, 0:12] - o.foot_forces()).max() <= 1e-8, e
        assert np.abs(aux[e, 12:18] - toe).max() <= 1e-8 and np.abs(aux[e, 18:24] - heel).max() <= 1e-8, e
        wq = split(oracle_row(o, m, names[:nbn], kinds[:nbn]), nbn)[0]
        assert np.abs(qa[e] - wq[:b.nv]).max() <= 1e-8 * np.abs(wq).max(), e
    for o in os_:
        o.close()
    b.close()


def test_aos_entry_point_equals_compact_path(P):
    """cassie_sim_step_pd_batch with contact rows == the compact path with the same rows and inputs, bit for bit"""
    n = 4096
    a, b = P.CassieBatch(n, precision=P.FP32), P.CassieBatch(n, precision=P.FP32)
    vals = batch_values('cassie', n, 300, base(a))
    for x in (a, b):
        x.set_env_contact(*vals)
    b.enable_estimator_device(True)
    pd = (P.pd_in_t * n)()
    for e in range(n):
        for side, leg in enumerate((pd[e].leftLeg, pd[e].rightLeg)):
            for i in range(5):
                leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
    _pd(P, b, n)
    for _ in range(200):
        a.step_pd(pd)
        b.step(1)
    assert np.array_equal(a.qpos(), b.qpos()) and np.array_equal(a.obs(), b.obs())
    a.close()
    b.close()


def test_rows_are_model_inputs(P, oracle_mod):
    """refusals change nothing; reset and snapshot restore keep the rows; a masked set changes only the masked rows; a device-pointer write takes
    effect at the next launch and get reports it; entries of visual geoms are ignored; the clear / carry-along interplay with mechanics rows"""
    import torch
    model, n = 'cassie_tray_box', 4
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    ref = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64)
    b0 = base(b)
    mc0 = b.env_mechanics()
    vals = batch_values(model, n, 20, b0)
    g = colliding(model)[2]
    visual = [x for x in range(len(b0[2])) if x not in colliding(model)]
    for x in visual:   # anything in a visual geom's entries is accepted and ignored
        vals[0][1:, x] = [np.nan, 1.0]
        vals[2][1:, x] = -1.0
    b.set_env_contact(*vals)
    got = b.env_contact()
    for k, v, m0 in zip(PARTS, vals, b0):   # get: the values given, the model's for visual geoms
        want = v.copy()
        want[:, visual] = m0[visual]
        assert np.array_equal(got[k], want), k
    vals = [got[k] for k in PARTS]
    assert all(np.array_equal(b.env_mechanics()[k], mc0[k]) for k in mc0)   # implicit mechanics rows hold the model's
    for part, idx, v in ((0, (2, g, 0), np.nan), (0, (1, g), [0.02, -1.0]), (1, (3, g, 1), 1.0), (1, (0, g, 4), 0.5), (2, (1, g), -0.5)):
        bad = [x.copy() for x in vals]
        bad[part][idx] = v
        with pytest.raises(RuntimeError, match='environment %d' % idx[0]):
            b.set_env_contact(*bad)
    assert all(np.array_equal(b.env_contact()[k], x) for k, x in zip(PARTS, vals))
    b.step(50)
    s = b.get_state()
    b.reset()
    b.set_state(s, mask=np.array([1, 0, 1, 0], dtype=np.uint8))
    assert all(np.array_equal(b.env_contact()[k], x) for k, x in zip(PARTS, vals))
    # a masked set changes the masked rows only
    dev = b.torch_view('contact')
    assert tuple(dev.shape) == (n, 256)
    before = dev.clone()
    sr = vals[0].copy()
    sr[:, g, 0] = 0.011
    b.set_env_contact(solref=sr, mask=np.array([0, 1, 0, 0], dtype=np.uint8))
    after = b.torch_view('contact')
    changed = (after != before).any(dim=1).cpu().numpy()
    assert list(changed) == [False, True, False, False]
    # a device write: a softer floor in environment 3, seen by get and by the next launch (against an oracle given it)
    floor_slot = int(np.flatnonzero((after[0].view(32, CT_SLOT)[:, CT_SOLREF] != 0).cpu().numpy())[0])
    rows = b.torch_view('contact')
    rows[3, CT_SLOT * floor_slot + CT_SOLREF] = 0.012
    torch.cuda.synchronize()
    got = b.env_contact()
    assert 0.012 in got['solref'][3][:, 0]
    b.reset()
    o = contact_oracle(oracle_mod, model, *[got[k][3] for k in PARTS])
    o.forward()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    _pd(P, b, n)
    for _ in range(300):
        b.step(1)
        o.step_pd(u)
    assert np.abs(b.qpos()[3, :o.nq] - o.arr('qpos')).max() <= 1e-9
    o.close()
    # clear: back to the model's values and to a batch that never had rows, bitwise (the implicit mechanics and actuator rows go too)
    b.clear_env_contact()
    assert not b.device_ptr('contact') and not b.device_ptr('mechanics') and not b.device_ptr('actuators')
    assert all(np.array_equal(b.env_contact()[k][0], x) for k, x in zip(PARTS, b0))
    for x in (b, ref):
        x.reset()
        _pd(P, x, n)
        x.step(50)
    assert np.array_equal(b.qpos(), ref.qpos()) and np.array_equal(b.obs(), ref.obs())
    # mechanics rows written after the contact rows stay when the contact rows go; clear_env_mechanics keeps model-valued rows under contact rows
    b.set_env_contact(*vals)
    arm = mc0['armature'].copy()
    arm[:, 6] *= 1.2
    b.set_env_mechanics(armature=arm)
    b.clear_env_contact()
    assert b.device_ptr('mechanics') and np.array_equal(b.env_mechanics()['armature'], arm)
    b.clear_env_mechanics()
    b.set_env_contact(*vals)
    b.clear_env_mechanics()
    assert b.device_ptr('mechanics') and all(np.array_equal(b.env_mechanics()[k], mc0[k]) for k in mc0)
    b.clear_env_contact()
    assert not b.device_ptr('mechanics')
    b.close()
    ref.close()


def test_legacy_simulator_and_copy(P, oracle_mod):
    """rows set on a simulator's batch: cassie_sim_step_pd follows the oracle with them, cassie_sim_copy copies them (the copy steps bit for bit as its
    source)"""
    O = oracle_mod
    L = P.lib()
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    dp = C.POINTER(C.c_double)
    L.cassie_batch_set_env_contact.argtypes = [C.c_void_p, dp, dp, dp, C.c_void_p]
    L.cassie_batch_set_env_contact.restype = C.c_int
    s1, s2 = (P.CassieSim(P.model_path('cassie')) for _ in range(2))
    probe = P.CassieBatch(1, modelfile=P.model_path('cassie'), precision=P.FP64)
    vals = random_contact('cassie', 5, base(probe))
    probe.close()
    arr = [np.ascontiguousarray(v[None], dtype=np.float64) for v in vals]
    assert L.cassie_batch_set_env_contact(L.cassie_sim_batch(s1.c), *[a.ctypes.data_as(dp) for a in arr], None) == 0
    o = contact_oracle(O, 'cassie', *vals)
    pin = P.pd_in_t()
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    C.memmove(C.addressof(pin), C.addressof(u), C.sizeof(pin))
    for _ in range(400):
        s1.step_pd(pin)
        o.step_pd(u)
    assert np.abs(s1.qpos() - o.arr('qpos')[:35]).max() <= 1e-9
    o.close()
    s2.copy(s1)
    for _ in range(200):
        s1.step_pd(pin)
        s2.step_pd(pin)
    assert np.array_equal(s1.qpos(), s2.qpos())
