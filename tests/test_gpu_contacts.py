"""GPU: contact lists (cassie_batch_enable_contacts, the F_CL instances) against the numpy restatement over the fp64 oracle
(tests/contact_list_support.py), the same batch on the F_FR chain twin, and the verb's rules: which launches write the rows, the device view,
the trace refusals, dropping the lists; and the model's name tables (cassie_batch_name2id / id2name)."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from contact_list_support import CON_HEAD, CON_SLOT, CON_W, FORCE, FRAME, GEOM1, GEOM2, POS, compare, restate, slots, table
from test_contacts import FP32_FORCE, FP32_GEO

pytestmark = pytest.mark.gpu
MODELS_ALL = ['cassie', 'cassie_depth', 'cassie_hfield', 'cassie_tray_box']


@pytest.fixture(scope='module')
def P():
    return product()


def _pd(P, b, n, rng=None):
    pt = np.tile(PD_TARGET, (n, 1))
    if rng is not None:
        pt = pt + rng.uniform(-0.05, 0.05, pt.shape)
    b.set_pd(P.pd_rows(n, pTarget=pt, pGain=PD_PGAIN, dGain=PD_DGAIN))


def _batch(P, model, prec, n):
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32 if prec == 'fp32' else P.FP64)
    b.enable_aux()
    b.enable_accelerations()
    return b


def _raw(b):
    out = np.zeros((b.n, CON_W))
    assert b._contacts_lib().cassie_batch_get_contacts(b.h, b._dp(out)) == 0
    return out


# ------------------------------------------------------------------ 1. against the oracle
@pytest.mark.parametrize('model', MODELS_ALL)
def test_four_fp64_envs_follow_the_oracle(P, oracle_mod, model):
    """fp64, 4 environments stepped like the oracle through stance and a fall, and a forward at the end: every environment's row against the
    restatement of the oracle's contacts -- counts, geoms, condim and efc addresses exact, geometry within 1e-9 and forces within 1e-7 of their scale
    (the trajectories drift apart by rounding: test_gpu_frames's bars)"""
    O = oracle_mod
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    t = table(model)
    b = _batch(P, model, 'fp64', 4)
    b.enable_contacts()
    _pd(P, b, 4)
    stance, off = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    listed = 0
    for k in range(10):
        if k == 5:
            b.set_pd(np.zeros((4, 52)))
        b.step(50)
        for _ in range(50):
            o.step_pd(stance if k < 5 else off)
        want = restate(o, t)
        got = _raw(b)
        for e in range(4):
            exact, geo, force = compare(got[e], want)
            assert exact and geo < 1e-9 and force < 1e-7, (model, k, e, exact, geo, force, got[e][:3], want[:3])
        listed = max(listed, int(want[0]))
    b.forward()
    o.forward()
    want, got = restate(o, t), _raw(b)
    exact, geo, force = compare(got[0], want)
    assert exact and geo < 1e-9 and force < 1e-7, (model, 'forward', geo, force)
    assert listed >= 2
    b.close()
    o.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield'])
def test_4096_fp32_envs_against_the_oracle(P, oracle_mod, model):
    """fp32, 4096 environments of configs 2 and 5 (cassie.xml stance; the height-field model), 64 sampled environments against the fp64 oracle at
    the fp32 bars of tests/test_contacts.py after 200 ticks of stance"""
    O = oracle_mod
    n = 4096
    b = _batch(P, model, 'fp32', n)
    b.enable_contacts()
    _pd(P, b, n)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    launches = 20 if model == 'cassie_hfield' else 4   # the height-field model's robot starts above the terrain
    for _ in range(launches):
        b.step(50)
    for _ in range(50 * launches):
        o.step_pd(u)
    want, got = restate(o, table(model)), _raw(b)
    worst = [0.0, 0.0]
    for e in np.random.default_rng(1).choice(n, 64, replace=False):
        exact, geo, force = compare(got[e], want)
        assert exact, (e, got[e][:3], want[:3])
        worst = [max(worst[0], geo), max(worst[1], force)]
    print(model, 'fp32 4096: geometry %.3g force %.3g' % tuple(worst))
    assert worst[0] < FP32_GEO and worst[1] < FP32_FORCE and want[0] >= 2, worst
    b.close()
    o.close()


# ------------------------------------------------------------------ 2. the twins change no physics
@pytest.mark.parametrize('prec', ['fp32', 'fp64'])
@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_twins_change_no_physics(P, model, prec):
    """64 environments with their own targets, single-tick and 50-tick launches through stance and a fall: qpos, qvel, obs, aux, acceleration rows
    and counters of the batch with contact lists equal those of the same batch on the chain twin (model-valued applied rows), bit for bit"""
    n = 64
    a, c = _batch(P, model, prec, n), _batch(P, model, prec, n)
    a.enable_contacts()
    c.enable_applied_forces()
    for x in (a, c):
        x.reset()
        _pd(P, x, n, np.random.default_rng(3))
    nk = 16 if model == 'cassie_hfield' else 4   # the height-field model's robot starts above the terrain
    for k in range(nk):
        if k == nk // 2:
            for x in (a, c):
                x.set_pd(np.zeros((n, 52)))
        for nt in (1, 50):
            a.step(nt)
            c.step(nt)
            for name in ('qpos', 'qvel', 'obs', 'aux', 'counters', 'qacc'):
                assert np.array_equal(getattr(a, name)(), getattr(c, name)()), (model, prec, k, nt, name)
    assert _raw(a)[:, 0].max() >= 2
    a.close()
    c.close()


# ------------------------------------------------------------------ 3. which launches write the rows
def test_launches_that_write_the_rows(P):
    """forward_where fills the masked environments only; reset_where, query, set_const, Jacobian, dynamics and inverse launches and set_state leave
    the rows alone; torch_view('contacts') is get_contacts' copy"""
    import torch
    n = 8
    b = _batch(P, 'cassie', 'fp64', n)
    b.set_frames(['left-foot'])
    b.enable_contacts()
    _pd(P, b, n, np.random.default_rng(2))
    snap = b.get_state()
    b.set_reset_bank(snap)
    b.step(100)
    rows = _raw(b)
    assert rows[:, 0].min() >= 1
    v = b.torch_view('contacts')
    b.sync()
    assert v.shape == (n, CON_W) and np.array_equal(v.cpu().numpy(), rows)
    b.query()
    b.set_const()
    b.frame_jacobian(0)
    b.compute_dynamics()
    b.compute_inverse(np.zeros((n, 32)))
    b.reset_where(torch.ones(n, dtype=torch.bool, device='cuda'))
    b.sync()
    assert np.array_equal(_raw(b), rows)
    mask = torch.zeros(n, dtype=torch.bool, device='cuda')
    mask[::2] = True
    b.forward_where(mask)
    b.sync()
    after = _raw(b)
    assert np.array_equal(after[1::2], rows[1::2])
    assert not np.array_equal(after[0::2], rows[0::2])   # restored to the start state, then listed again
    b.set_state(snap)
    assert np.array_equal(_raw(b), after)
    b.close()


# ------------------------------------------------------------------ 4. refusals and dropping the lists
def test_trace_and_contacts_refuse_each_other_and_dropping_returns(P):
    n = 64
    a, b, c, d = (_batch(P, 'cassie', 'fp32', n) for _ in range(4))
    a.enable_contacts()
    with pytest.raises(RuntimeError, match='trace'):
        a.set_trace([(0, 2)], 10)
    c.set_trace([(0, 2)], 10)
    with pytest.raises(RuntimeError, match='trace'):
        c.enable_contacts()
    c.set_trace([])
    c.enable_contacts()
    d.enable_applied_forces()
    for x in (a, b, c, d):
        x.reset()
        _pd(P, x, n, np.random.default_rng(5))
        x.step(50)
    a.enable_contacts(False)
    c.enable_contacts(False)
    d.enable_applied_forces(False)
    for x in (a, b, c, d):
        x.step(50)
    for name in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
        assert np.array_equal(getattr(a, name)(), getattr(b, name)()), name
        assert np.array_equal(getattr(c, name)(), getattr(d, name)()), name
    assert not a.device_ptr('applied') and not a.device_ptr('contacts')
    with pytest.raises(RuntimeError):
        a.contacts()
    for x in (a, b, c, d):
        x.close()


# ------------------------------------------------------------------ 5. the contact-Jacobian recipe
def test_contact_jacobian_recipe(P, oracle_mod):
    """fp64, standing: the normal row of each listed contact built from the two bodies' frame Jacobians, Jp(b, p) = jacp(b) - [p - xpos(b)]x jacr(b)
    projected on the frame's normal, equals the oracle's efc_J normal row (the mean of the contact's first two pyramid rows) within 1e-10"""
    O = oracle_mod
    model = 'cassie'
    t = table(model)
    body = [int(x) for x in t['geom_bodyid']]
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    b = _batch(P, model, 'fp64', 1)
    b.set_frames(list(t['names_body']))
    b.enable_contacts()
    _pd(P, b, 1)
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for _ in range(200):
        o.step_pd(u)
    b.step(200)
    o.forward()
    b.forward()
    row = _raw(b)[0]
    fr = b.frames()[0]
    J = o.efc_J()
    s = slots(row)
    n = 0
    for c in range(int(row[0])):
        p, nrm = s[c, POS:POS + 3], s[c, FRAME:FRAME + 3]
        jn = np.zeros(o.nv)
        for g, sign in ((int(s[c, GEOM1]), -1), (int(s[c, GEOM2]), 1)):
            bi = body[g]
            if bi == 0:
                continue
            jp, jr = b.frame_jacobian(bi)
            jp, jr = jp[0], jr[0]
            r = p - fr[bi, 0:3]
            jpp = jp - np.cross(r, jr.T).T
            jn += sign * nrm @ jpp
        e0 = int(s[c, 23])
        want = 0.5 * (J[e0] + J[e0 + 1])
        assert np.abs(jn - want).max() < 1e-10 * max(1.0, np.abs(want).max()), c
        n += 1
    assert n >= 2
    b.close()
    o.close()


# ------------------------------------------------------------------ 6. names
@pytest.mark.parametrize('model', MODELS_ALL + ['cassie_mass', 'cassie_no_grav'])
def test_names_round_trip(P, model):
    """every named body, joint, geom, site and camera of the model table resolves to its index and back; unknown names and kinds give -1 / None;
    the legacy cassie_sim_mj_name2id agrees"""
    t = {ln.split()[0]: ln.split()[3:] for ln in open(P.model_path(model)).read().split('\n') if ln.strip()}   # the compiled table the batch loads
    if os.path.exists(os.path.join(GOLDEN, model + '.omodel')):   # the oracle's numbering
        assert all(t[k] == table(model)[k] for k in ('names_body', 'names_joint', 'names_geom', 'names_site'))
    b = P.CassieBatch(1, modelfile=P.model_path(model), precision=P.FP64)
    for kind, key in (('body', 'names_body'), ('xbody', 'names_body'), ('joint', 'names_joint'), ('geom', 'names_geom'), ('site', 'names_site'),
                      ('camera', 'names_camera')):
        names = [x if x != '-' else '' for x in t.get(key, [])]
        for i, nm in enumerate(names):
            if nm:
                assert b.name2id(kind, nm) == i and b.id2name(kind, i) == nm, (kind, nm, i)
            else:
                assert b.id2name(kind, i) is None
        assert b.id2name(kind, len(names)) is None and b.id2name(kind, -1) is None
        assert b.name2id(kind, 'no-such-object') == -1
    for kind in ('actuator', 'equality', 'mesh', 'dof', 'nonsense'):
        assert b.name2id(kind, 'left-foot') == -1 and b.id2name(kind, 0) is None
    b.close()
    s = P.CassieSim(P.model_path(model))
    assert s.mj_name2id('body', 'left-foot') == t['names_body'].index('left-foot')
    assert s.mj_name2id('geom', 'no-such-geom') == -1 and s.mj_name2id('actuator', 'x') == -1
