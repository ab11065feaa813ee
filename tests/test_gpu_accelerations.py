"""GPU: acceleration rows (cassie_batch_enable_accelerations) -- the F_FR kernel instances' accel_row against one oracle per sampled environment, bitwise
neutrality for every other output, snapshots, the zero-copy view and the legacy verbs.  CPU twins (host emulation): tests/test_accelerations.py."""
import os
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_accelerations import oracle_row, restate, split
from test_frames import all_frames, omodel
from test_gpu_frames import _jitter, _pd_in, _rows

pytestmark = pytest.mark.gpu

MODELS = os.path.join(os.path.dirname(GOLDEN), '..', 'cassie-mujoco-sim_b200', 'models')
EIGHT = ['cassie-pelvis', 'left-hip-pitch', 'left-shin', 'left-foot', 'right-hip-pitch', 'right-tarsus', 'right-foot', 'right-toe']
EIGHT_KINDS = [0, 0, 0, 0, 0, 0, 0, 1]


def _frames(model, which):
    if which == 'all':
        return all_frames(model)
    names, kinds = list(EIGHT), list(EIGHT_KINDS)
    if model == 'cassie_tray_box':   # the cup instead of the right hip pitch, and the model's one site
        m = omodel(model)
        names[4], names[7] = m['names_body'][-1], m['names_site'][0]
    return names, kinds


def _batch(P, model, n, fp64, names, kinds):
    b = P.CassieBatch(n, modelfile=os.path.join(MODELS, model + '.cmodel'), precision=P.FP64 if fp64 else P.FP32)
    b.set_frames(names, kinds)
    b.enable_accelerations(True)
    q = b.qpos() + _jitter(n, b.qpos().shape[1])
    b.set_qpos(q)
    b.set_pd(_rows(P, n, True))
    b.forward()
    return b, q


def _row(b, e, nf):
    """environment e's acceleration row as the emulation lays it out (qacc padded to 40, slots of 8)"""
    r = np.zeros(40 + 8 * nf)
    r[:b.nv] = b.qacc()[e]
    r[40:].reshape(nf, 8)[:, :6] = b.body_accelerations()[e]
    return r


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
@pytest.mark.parametrize('which', ['eight', 'all'])
def test_fp64_accelerations_follow_the_oracle(oracle_mod, model, which):
    """256 fp64 environments through a stance and a fall; 64 sampled ones replayed by the oracle: qacc and cacc within 1e-8 of the largest magnitude"""
    O, P = oracle_mod, product()
    n, nsample, ticks, every = 256, 64, 300, 50
    names, kinds = _frames(model, which)
    b, q = _batch(P, model, n, True, names, kinds)
    m = omodel(model)
    sample = np.random.default_rng(5).choice(n, nsample, replace=False)
    oracles = []
    for e in sample:
        o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
        o.arr('qpos')[:] = q[e, :o.nq]
        o.forward()
        oracles.append(o)
    stance, motors_off = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    worst, scale = dict(qacc=0.0, cacc=0.0), dict(qacc=0.0, cacc=0.0)
    for k in range(ticks):
        if k == ticks // 2:
            b.set_pd(_rows(P, n, False))
        b.step(1)
        for o in oracles:
            o.step_pd(stance if k < ticks // 2 else motors_off)
        if k % every == every - 1:
            qa, ca = b.qacc(), b.body_accelerations()
            for e, o in zip(sample, oracles):
                wq, wc, _ = split(oracle_row(o, m, names, kinds), len(names))
                worst['qacc'] = max(worst['qacc'], np.abs(qa[e] - wq[:b.nv]).max())
                worst['cacc'] = max(worst['cacc'], np.abs(ca[e] - wc).max())
                scale['qacc'] = max(scale['qacc'], np.abs(wq).max())
                scale['cacc'] = max(scale['cacc'], np.abs(wc).max())
    print(model, which, worst, scale)
    assert worst['qacc'] <= 1e-8 * scale['qacc'] and worst['cacc'] <= 1e-8 * scale['cacc'], (worst, scale)


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
@pytest.mark.parametrize('which', ['eight', 'all'])
def test_fp32_accelerations_at_the_oracle_state(oracle_mod, model, which):
    """4096 fp32 environments stepped through a stance; then a forward launch, and 64 sampled environments against a fresh oracle placed at the same
    state (qpos, qvel, warm start = the step's qacc; zero ctrl): within 1e-2 of the largest magnitude, or of 20 m/s^2 (the single-precision solve of the
    closed-chain rows, tests/test_accelerations.py)"""
    O, P = oracle_mod, product()
    n = 4096
    names, kinds = _frames(model, which)
    b, _ = _batch(P, model, n, False, names, kinds)
    m = omodel(model)
    sample = np.random.default_rng(6).choice(n, 64, replace=False)
    worst = 0.0
    for k in range(3):
        b.step(100)
        q, v, ws = b.qpos(), b.qvel(), b.qacc()
        b.forward()
        for e in sample:
            o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
            o.arr('qpos')[:] = q[e, :o.nq]
            o.arr('qvel')[:] = v[e]
            o.arr('qacc_warmstart')[:] = ws[e]
            o.forward()
            gq, gc, _ = split(_row(b, e, len(names)), len(names))
            wq, wc, _ = split(oracle_row(o, m, names, kinds), len(names))
            worst = max(worst, np.abs(gq - wq).max() / max(20.0, np.abs(wq).max()), np.abs(gc - wc).max() / max(20.0, np.abs(wc).max()))
            o.close()
    print(model, which, worst)
    assert worst <= 1e-2


@pytest.mark.parametrize('fp64', [True, False])
def test_accelerations_change_no_other_output(fp64):
    """1000 ticks with and without acceleration rows (both with 8 frames): qpos, qvel, obs, aux, frames and the counters bitwise equal; and a batch
    with acceleration rows but no frames against the shipped extended instance"""
    P = product()
    n = 256
    a, b, c, d = (P.CassieBatch(n, precision=P.FP64 if fp64 else P.FP32) for _ in range(4))
    for x in (a, b):
        x.set_frames(EIGHT, EIGHT_KINDS)
    b.enable_accelerations(True)
    d.enable_accelerations(True)
    for x in (a, b, c, d):
        x.enable_aux(True)
        x.set_qpos(x.qpos() + _jitter(n, x.qpos().shape[1]))
        x.set_pd(_rows(P, n, True))
        x.forward()
    for k in range(1000):
        if k == 500:
            for x in (a, b, c, d):
                x.set_pd(_rows(P, n, False))
        for x in (a, b, c, d):
            x.step(1)
        if k % 50 == 49:
            for f in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
                assert np.array_equal(getattr(a, f)(), getattr(b, f)()), (k, f)
                assert np.array_equal(getattr(c, f)(), getattr(d, f)()), (k, f)
            assert np.array_equal(a.frames(), b.frames()), k
    assert np.abs(b.qacc()).max() > 1 and np.abs(d.qacc()).max() > 1 and d.body_accelerations().shape == (n, 0, 6)


def test_snapshot_restores_rows_and_torch_view():
    import torch
    P = product()
    n = 64
    b, _ = _batch(P, 'cassie_tray_box', n, False, *_frames('cassie_tray_box', 'eight'))
    b.step(50)
    snap = b.get_state()
    qa, ca = b.qacc(), b.body_accelerations()
    b.step(50)
    assert not np.array_equal(qa, b.qacc())
    b.set_state(snap)
    assert np.array_equal(qa, b.qacc()) and np.array_equal(ca, b.body_accelerations())
    mask = (np.arange(n) % 2 == 0).astype(np.uint8)
    b.step(5)
    after = b.qacc()
    b.set_state(snap, mask=mask)
    got = b.qacc()
    assert np.array_equal(got[mask == 1], qa[mask == 1]) and np.array_equal(got[mask == 0], after[mask == 0])
    b.sync()
    v = b.torch_view('acc')
    assert tuple(v.shape) == (n, 40 + 8 * 8) and v.dtype == torch.float32
    rows = v.cpu().numpy().astype(np.float64)
    assert np.array_equal(rows[:, :b.nv], b.qacc()) and np.array_equal(rows[:, 40:].reshape(n, 8, 8)[:, :, :6], b.body_accelerations())
    b.free_state(snap)


def test_api_edges():
    P = product()
    b = P.CassieBatch(8, precision=P.FP32)
    with pytest.raises(RuntimeError):
        b.qacc()
    b.enable_accelerations(True)
    assert b.row_width('acc') == 40 and not b.qacc().any()
    b.step(2)
    assert np.abs(b.qacc()).max() > 0
    b.set_frames(['world', 'cassie-pelvis', 'left-toe'], [0, 0, 1])
    assert b.row_width('acc') == 64 and not b.qacc().any() and b.body_accelerations().shape == (8, 3, 6)
    b.reset()
    ca = b.body_accelerations()
    assert np.allclose(ca[:, 0], [0, 0, 0, 0, 0, 9.81]) and not ca[:, 2].any() and np.abs(ca[:, 1]).max() > 0   # the reset's forward fills them
    b.enable_accelerations(False)
    with pytest.raises(RuntimeError):
        b.body_accelerations()
    with pytest.raises(RuntimeError):
        b.torch_view('acc')
    b.step(2)


def _model_with_foot_middle(tmp):
    """cassie.cmodel with its right-foot-pt site named right-foot-middle (the site the reference's foot_orient reads; the shipped models name it
    differently)"""
    src = open(os.path.join(MODELS, 'cassie.cmodel')).read()
    path = os.path.join(tmp, 'cassie_foot_middle.cmodel')
    with open(path, 'w') as f:
        f.write(src.replace(' right-foot-pt ', ' right-foot-middle '))
    return path


def test_legacy_acceleration_verbs_follow_the_oracle(oracle_mod):
    """CassieSim.qacc(), get_body_acceleration (every body) and foot_quat through a stance against the oracle; after full_reset qacc is zero and
    every body reads (0, 0, 0, -g); a state restore brings the rows back; an unknown body reads zeros"""
    P, O = product(), oracle_mod
    m = omodel('cassie')
    bodies = list(m['names_body'])
    with tempfile.TemporaryDirectory() as tmp:
        c = P.CassieSim(_model_with_foot_middle(tmp))
        o = O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
        pu, u = _pd_in(P), O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
        worst = dict(qacc=0.0, cacc=0.0, quat=0.0)
        for k in range(300):
            c.step_pd(pu)
            o.step_pd(u)
            if k % 50 == 49:
                _, _, cacc = restate(m, o.arr('cdof'), o.arr('qvel').copy(), o.arr('qacc').copy())
                worst['qacc'] = max(worst['qacc'], np.abs(c.qacc() - o.arr('qacc')).max() / np.abs(o.arr('qacc')).max())
                for bi, name in enumerate(bodies):
                    a = np.zeros(6)
                    c.get_body_acceleration(a, name)
                    worst['cacc'] = max(worst['cacc'], np.abs(a - cacc[bi]).max() / np.abs(cacc).max())
                quat = np.zeros(4)
                c.foot_quat(quat)
                assert np.array_equal(quat, np.array(c.get_site_quat('right-foot-middle')))
                assert np.abs(quat).max() > 0.1
        print(worst)
        assert worst['qacc'] <= 1e-8 and worst['cacc'] <= 1e-8
        s = c.get_state()
        keep = c.qacc()
        for _ in range(20):
            c.step_pd(pu)
        assert not np.array_equal(keep, c.qacc())
        c.set_state(s)
        assert np.array_equal(keep, c.qacc())
        c.full_reset()
        assert not c.qacc().any()
        for name in bodies:
            a = np.zeros(6)
            c.get_body_acceleration(a, name)
            assert np.array_equal(a, [0, 0, 0, 0, 0, 9.81]), name
        a = np.ones(6)
        c.get_body_acceleration(a, 'no-such-body')
        assert not a.any()
    plain = P.CassieSim()   # the shipped cassie.xml has no right-foot-middle site: zeros, like an unknown site
    quat = np.ones(4)
    plain.foot_quat(quat)
    assert not quat.any()
