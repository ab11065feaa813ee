"""GPU: per-tick traces of multi-tick launches (cassie_batch_set_trace, the F_TC instances), against the rows single-tick launches leave, the same
batch without a trace, the fp64 oracle tick by tick, and the verb's rules: refusals, slots, trace_ticks, the device view, cassie_sim_step_pd_batch."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_gpu_configs import BARS

pytestmark = pytest.mark.gpu

QPOS, QVEL, OBS, AUX, FRAME = range(5)
# (model, precision, extra rows, the instance step_entry routes the traced batch to), as test_gpu_env_contact.py's ROUTES
ROUTES = [('cassie', 'fp32', None, 'f1fc4'), ('cassie', 'fp32', 'frames', 'f1fd7'), ('cassie', 'fp64', None, 'd1fd7'), ('cassie', 'fp32', 'geom', 'f1fdf'),
          ('cassie', 'fp64', 'geom', 'd1fdf'), ('cassie_hfield', 'fp32', 'hfield', 'f1fff'), ('cassie_hfield', 'fp64', 'hfield', 'd1fff')]


@pytest.fixture(scope='module')
def P():
    return product()


def _pd(P, b, n, rng=None):
    pt = np.tile(PD_TARGET, (n, 1))
    if rng is not None:
        pt = pt + rng.uniform(-0.05, 0.05, pt.shape)   # every environment its own targets
    b.set_pd(P.pd_rows(n, pTarget=pt, pGain=PD_PGAIN, dGain=PD_DGAIN))


def _batch(P, model, prec, extra, n):
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP32 if prec == 'fp32' else P.FP64)
    b.enable_aux()
    if extra == 'frames':
        b.set_frames(['left-foot', 'right-foot', 'cassie-pelvis'])
    elif extra == 'geom':
        b.set_env_geom_pose('floor', pos=[0.0, 0.0, 0.0])
    elif extra == 'hfield':
        b.set_env_hfield(terrain=0)
    return b


def _columns(b, frames):
    cols = [(QPOS, c) for c in (0, 1, 2, 3, 6, 10)] + [(QVEL, c) for c in (0, 2, 5, 20, 31)]
    cols += [(OBS, c) for c in (0, 9, 20, 29, 42, 46, 55, 56, 60, 75, 86)]
    cols += [(AUX, c) for c in (0, 2, 8, 14, 20, 24, 26, 29, 30, 33, 42, 45, 48, 51, 54)]
    if frames:
        cols += [(FRAME, c) for c in (0, 2, 3, 6, 9, 15, 20, 42, 45, 59)]
    return cols


def _rows(b, cols, frames):
    """the traced columns as cassie_batch_get_* returns them now: [n, k]"""
    src = {QPOS: b.qpos(), QVEL: b.qvel(), OBS: b.obs(), AUX: b.aux()}
    if frames:
        src[FRAME] = b.frames().reshape(b.n, -1)
    return np.stack([src[s][:, c] for s, c in cols], axis=1)


# ------------------------------------------------------------------ 1. one 50-tick launch is 50 single-tick launches, and the physics of the twin
@pytest.mark.parametrize('model,prec,extra,tag', ROUTES, ids=[r[3] for r in ROUTES])
def test_trace_is_single_tick_rows_and_changes_no_physics(P, model, prec, extra, tag):
    """64 environments with their own targets, 4 launches of 50 ticks (stance, then a fall): the trace equals the rows read after each of 50
    single-tick launches of a second batch, bit for bit; qpos, qvel, obs, aux and the counters of the traced batch equal, bit for bit, those of the
    same batch with model-valued applied rows and no trace (the chain twin)"""
    n = 64
    frames = extra == 'frames'
    a, b, c = (_batch(P, model, prec, extra, n) for _ in range(3))
    cols = _columns(a, frames)
    a.set_trace(cols, 50)
    b.set_trace(cols, 50)
    c.enable_applied_forces()
    for x in (a, b, c):
        x.reset()
        _pd(P, x, n, np.random.default_rng(3))
    for k in range(4):
        if k == 2:
            for x in (a, b, c):
                x.set_pd(np.zeros((n, 52)))
        a.step(50)
        c.step(50)
        want = []
        for t in range(50):
            b.step(1)
            want.append(_rows(b, cols, frames))
        assert b.trace_ticks() == 1 and a.trace_ticks() == 50
        got, want = a.trace(), np.stack(want, axis=1)
        bad = np.argwhere(got != want)
        assert bad.size == 0, (tag, k, [(int(e), int(t), cols[int(i)]) for e, t, i in bad[:8]])
        for name in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
            assert np.array_equal(getattr(a, name)(), getattr(c, name)()), (tag, k, name)
    for x in (a, b, c):
        x.close()


# ------------------------------------------------------------------ 2. against the oracle
def test_four_envs_fp64_follow_the_oracle(P, oracle_mod):
    """fp64, 4 environments, 10 launches of 50 ticks: per tick qpos within 1e-9 (test_gpu_applied_forces's bar), foot / toe / heel forces within 1e-8,
    foot positions within 1e-10 and velocities within 1e-8 (test_derived's check_row), the centre of mass and the pelvis frame's xquat within 1e-10 of
    the state the tick started from (the rows describe it)"""
    O, n = oracle_mod, 4
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.enable_aux()
    b.set_frames(['cassie-pelvis'])
    cols = [(QPOS, c) for c in range(7)] + [(AUX, c) for c in range(45)] + [(FRAME, 3 + i) for i in range(4)]
    b.set_trace(cols, 50)
    b.reset()
    _pd(P, b, n)
    o = O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    o.set_caps()
    stance, off = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    worst = dict(qpos=0.0, force=0.0, pos=0.0, vel=0.0, cm=0.0, quat=0.0)
    for k in range(10):
        if k == 5:
            b.set_pd(np.zeros((n, 52)))
        b.step(50)
        tr = b.trace()
        for t in range(50):
            cm, quat = o.cm_position(), o.arr('xquat')[4:8].copy()
            o.step_pd(stance if k < 5 else off)
            toe, heel = o.heeltoe_forces()
            r = tr[:, t]
            worst['qpos'] = max(worst['qpos'], np.abs(r[:, :7] - o.arr('qpos')[:7]).max())
            a = r[:, 7:]
            worst['force'] = max(worst['force'], np.abs(a[:, 0:12] - o.foot_forces()).max(), np.abs(a[:, 12:18] - toe).max(), np.abs(a[:, 18:24] - heel).max())
            worst['pos'] = max(worst['pos'], np.abs(a[:, 24:30] - o.foot_positions()).max())
            worst['vel'] = max(worst['vel'], np.abs(a[:, 30:42] - o.foot_velocities()).max())
            worst['cm'] = max(worst['cm'], np.abs(a[:, 42:45] - cm).max())
            worst['quat'] = max(worst['quat'], np.abs(r[:, 52:56] - quat).max())
    print(worst)
    assert worst['qpos'] < 1e-9 and worst['force'] < 1e-8 and worst['pos'] < 1e-10 and worst['vel'] < 1e-8, worst
    assert worst['cm'] < 1e-10 and worst['quat'] < 1e-10, worst
    assert o.arr('qpos')[2] < 0.95
    b.close()
    o.close()


def test_fp32_4096_sampled_envs_follow_the_oracle(P, oracle_mod):
    """fp32, 4096 environments with their own targets, 6 launches of 50 ticks: the traced qpos of 16 sampled environments against the fp64 oracle every
    tick, median / 90th percentile / worst environment within configuration 2's bars"""
    O, n = oracle_mod, 4096
    rng = np.random.default_rng(11)
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    b.enable_aux()
    b.set_trace([(QPOS, c) for c in range(35)] + [(AUX, c) for c in range(12)], 50)
    b.reset()
    pt = np.tile(PD_TARGET, (n, 1)) + rng.uniform(-0.05, 0.05, (n, 10))
    b.set_pd(P.pd_rows(n, pTarget=pt, pGain=PD_PGAIN, dGain=PD_DGAIN))
    envs = rng.choice(n, 16, replace=False)
    os_ = [O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel')) for _ in envs]
    for o in os_:
        o.set_caps()
    us = [O.make_pd(pTarget=pt[e], pGain=PD_PGAIN, dGain=PD_DGAIN) for e in envs]
    err = np.zeros(len(envs))
    for k in range(6):
        b.step(50)
        tr = b.trace()
        for t in range(50):
            for i, (o, u) in enumerate(zip(os_, us)):
                o.step_pd(u)
                err[i] = max(err[i], np.abs(tr[envs[i], t, :35] - o.arr('qpos')).max())
    med, p90, worst = float(np.median(err)), float(np.percentile(err, 90)), float(err.max())
    print('4096 fp32 traced qpos: median %.1e, p90 %.1e, worst %.1e' % (med, p90, worst))
    assert med <= BARS[2][0] and p90 <= BARS[2][1] and worst <= BARS[2][2], (med, p90, worst)
    b.close()
    for o in os_:
        o.close()


# ------------------------------------------------------------------ 3. the verb's rules
def test_refusals_slots_and_views(P):
    import torch
    n = 8
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    L = b._trace_lib()

    def refused(cols, T=10, why=''):
        with pytest.raises(RuntimeError) as e:
            b.set_trace(cols, T)
        assert why in str(e.value), str(e.value)

    refused([(7, 0)], why='unknown source')
    refused([(QPOS, 35)], why='qpos column 35')
    refused([(QVEL, 32)], why='qvel column 32')
    refused([(OBS, 112)], why='observation column 112')
    refused([(QPOS, -1)])
    refused([(QPOS, 0)] * 65, why='between 0 and 64')
    refused([(QPOS, 0)], T=0, why='max_ticks')
    refused([(AUX, 0)], why='cassie_batch_enable_aux')
    refused([(FRAME, 0)], why='cassie_batch_set_frames')
    b.enable_aux()
    refused([(AUX, 64)], why='derived-quantity column 64')
    b.set_frames(['left-foot'])
    refused([(FRAME, 20)], why='frame column 20')
    assert not b.device_ptr('trace') and not b.device_ptr('applied')   # nothing changed
    # a trace of aux and frame columns pins those rows
    b.set_trace([(AUX, 2), (FRAME, 2), (QPOS, 2)], 8)
    assert b.device_ptr('applied') and b.device_ptr('contact')   # the twin's rows, allocated by set_trace
    with pytest.raises(RuntimeError, match='traced column'):
        b.enable_aux(False)
    with pytest.raises(RuntimeError, match='traced column'):
        b.set_frames(['right-foot'])
    assert b.trace_ticks() == 0
    # slots: nticks > T keeps the last T ticks; nticks < T writes 0 .. nticks - 1 and leaves the rest; other launches write nothing
    ref = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    ref.enable_aux()
    ref.set_frames(['left-foot'])
    ref.set_trace([(AUX, 2), (FRAME, 2), (QPOS, 2)], 50)
    for x in (b, ref):
        x.reset()
        _pd(P, x, n)
        x.step(50)
    assert b.trace_ticks() == 8 and np.array_equal(b.trace(), ref.trace()[:, 42:])
    before = b.trace()
    for x in (b, ref):
        x.step(5)
    assert b.trace_ticks() == 5
    view = b.torch_view('trace')
    assert tuple(view.shape) == (n, 8, 3)
    b.sync()
    full = view.cpu().numpy().astype(np.float64)
    assert np.array_equal(full[:, :5], ref.trace()[:, :5]) and np.array_equal(full[:, 5:], before[:, 5:])
    assert np.array_equal(b.trace(), full[:, :5])
    assert L.cassie_batch_row_width(b.h, b'trace') == 24
    b.forward()
    b.query()
    b.reset()
    b.set_state(b.get_state())
    assert np.array_equal(b.torch_view('trace').cpu().numpy().astype(np.float64), full)   # outputs only: nothing but a step writes them
    # cassie_sim_step_pd_batch records its one tick in slot 0
    pd = (P.pd_in_t * n)()
    b.step_pd(pd)
    got = b.trace()
    assert b.trace_ticks() == 1 and got.shape == (n, 1, 3) and np.array_equal(got[:, 0, 2], b.qpos()[:, 2])
    # the batch of a legacy simulator is refused
    sim = P.CassieSim(P.model_path('cassie'))
    b.L.cassie_sim_batch.restype = C.c_void_p
    b.L.cassie_sim_batch.argtypes = [C.c_void_p]
    sb = b.L.cassie_sim_batch(sim.c)
    one = (C.c_int * 1)(0)
    assert L.cassie_batch_set_trace(sb, one, one, 1, 4) == -1 and 'cassie_sim_t' in P._last_error()
    # k = 0 drops the trace and the rows it brought
    b.set_trace([])
    assert not b.device_ptr('trace') and not b.device_ptr('applied') and not b.device_ptr('contact')
    b.enable_aux(False)
    for x in (b, ref):
        x.close()
    torch.cuda.synchronize()


def test_dropping_the_trace_returns_to_the_untraced_instance(P):
    """set_trace then k = 0 runs what a batch never traced runs, bit for bit; a batch traced for a while, then dropped, follows one that had zeroed
    applied rows for the same while, bit for bit"""
    n = 64
    a, b, c, d = (_batch(P, 'cassie', 'fp32', None, n) for _ in range(4))
    a.set_trace([(QPOS, 2), (AUX, 2)], 10)
    a.set_trace([])
    c.set_trace([(QPOS, 2), (AUX, 2)], 10)
    d.enable_applied_forces()
    for x in (a, b, c, d):
        x.reset()
        _pd(P, x, n, np.random.default_rng(5))
        x.step(50)
    c.set_trace([])
    d.enable_applied_forces(False)
    for x in (a, b, c, d):
        x.step(50)
    for name in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
        assert np.array_equal(getattr(a, name)(), getattr(b, name)()), name
        assert np.array_equal(getattr(c, name)(), getattr(d, name)()), name
    assert not a.device_ptr('applied') and not c.device_ptr('applied')
    for x in (a, b, c, d):
        x.close()
