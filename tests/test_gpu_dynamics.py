"""GPU: dynamics rows (cassie_batch_dynamics, launch mode 5) -- the F_FR kernel instances against one oracle per sampled environment, with
per-environment constants, bitwise neutrality for stepping, the legacy verbs and the API's behaviour.  CPU twins (host emulation):
tests/test_dynamics.py."""
import os

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_dynamics import centroid, oracle_dynamics
from test_frames import all_frames, omodel

pytestmark = pytest.mark.gpu

MODELS = os.path.join(os.path.dirname(GOLDEN), '..', 'cassie-mujoco-sim_b200', 'models')


def _jitter(n, nq, seed=11):
    rng = np.random.default_rng(seed)
    d = np.zeros((n, nq))
    d[:, 0:2] = rng.uniform(-0.03, 0.03, (n, 2))
    d[:, 2] = rng.uniform(0, 0.02, n)
    if nq > 35:
        d[:, 35:38] = d[:, 0:3]
    return d


def _batch(model, fp64, n):
    P = product()
    b = P.CassieBatch(n, modelfile=os.path.join(MODELS, model + '.cmodel'), precision=P.FP64 if fp64 else P.FP32)
    b.set_qpos(b.qpos() + _jitter(n, b.qpos().shape[1]))
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.forward()
    return P, b


def _parity(O, model, fp64, n=256, nsample=32, consts=None):
    P, b = _batch(model, fp64, n)
    if consts:
        for k, v in consts.items():
            b.set_model(k, v)
        b.set_const()
    sample = np.random.default_rng(5).choice(n, nsample, replace=False)
    err = dict(M=0.0, bias=0.0, J_eq=0.0, eq_err=0.0, rcm=0.0, Icm=0.0)
    scale = dict(err)
    for phase in range(4):   # stance, stance, fall, fall
        if phase == 2:
            b.set_pd(P.pd_rows(n))
        b.step(100)
        b.compute_dynamics()
        got = b.dynamics()
        rcm = b.torch_view('dyn').cpu().numpy()[:, P.DYN['rcm']].astype(np.float64)
        q, v = b.qpos(), b.qvel()
        for e in sample:
            c = {k: vals[e] for k, vals in consts.items()} if consts else None
            want = oracle_dynamics(O, model, q[e], v[e], c)
            mine = dict(M=got['M'][e], bias=got['bias'][e], J_eq=got['J_eq'][e], eq_err=got['eq_err'][e], rcm=rcm[e], Icm=got['Icm'][e])
            assert np.allclose(mine['Icm'], centroid(mine['M'], mine['rcm']), rtol=0, atol=1e-9 * np.abs(mine['Icm']).max())   # the host helper
            for key in err:
                err[key] = max(err[key], np.abs(mine[key] - want[key]).max())
                scale[key] = max(scale[key], np.abs(want[key]).max())
    b.close()
    return err, scale


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_fp64_dynamics_follow_the_oracle(oracle_mod, model):
    err, scale = _parity(oracle_mod, model, True)
    print(model, err, scale)
    assert err['M'] <= 1e-12 * scale['M'] and err['J_eq'] <= 1e-12 * scale['J_eq'], (err, scale)
    assert err['bias'] <= 1e-10 * scale['bias'] and err['eq_err'] <= 1e-12, (err, scale)
    assert err['rcm'] <= 1e-12 and err['Icm'] <= 1e-12 * scale['Icm'], (err, scale)


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_fp32_dynamics_follow_the_oracle(oracle_mod, model):
    err, scale = _parity(oracle_mod, model, False)
    print(model, err, scale)
    for key in ('M', 'bias', 'J_eq', 'Icm'):
        assert err[key] <= 1e-4 * scale[key], (key, err, scale)
    assert err['eq_err'] <= 1e-5 and err['rcm'] <= 1e-5, (err, scale)


def test_dynamics_with_domain_randomisation(oracle_mod):
    n = 256
    m = omodel('cassie')
    rng = np.random.default_rng(9)
    consts = dict(body_mass=m['body_mass'] * rng.uniform(0.8, 1.2, (n, m['body_mass'].size)),
                  body_ipos=m['body_ipos'] + rng.uniform(-0.01, 0.01, (n, m['body_ipos'].size)),
                  dof_damping=m['dof_damping'] * rng.uniform(0.5, 1.5, (n, m['dof_damping'].size)))
    err, scale = _parity(oracle_mod, 'cassie', True, n=n, nsample=16, consts=consts)
    print(err, scale)
    assert err['M'] <= 1e-12 * scale['M'] and err['bias'] <= 1e-10 * scale['bias'] and err['rcm'] <= 1e-12, (err, scale)


@pytest.mark.parametrize('fp64,frames,env_geoms', [(False, False, False), (True, False, False), (False, True, False), (True, True, False),
                                                   (False, True, True), (True, False, True)])
def test_stepping_is_undisturbed(fp64, frames, env_geoms):
    """a batch that asks for the dynamics every 10 ticks stays bitwise equal to one that never asks, over 500 ticks (stance, then a fall)"""
    n = 128
    out = []
    for ask in (False, True):
        P, b = _batch('cassie', fp64, n)
        if frames:
            b.set_frames(*all_frames('cassie'))
            b.enable_aux(True)
        if env_geoms:
            b.set_env_geom_pose('box1', pos=[0.05, 0.135, 0.04 - 0.1], size=[0.25, 0.1, 0.1], mask=(np.arange(n) % 2 == 0).astype(np.uint8))
        for k in range(500):
            if k == 250:
                b.set_pd(P.pd_rows(n))
            b.step(1)
            if ask and k % 10 == 0:
                b.compute_dynamics()
        rec = dict(qpos=b.qpos(), qvel=b.qvel(), obs=b.obs(), counters=b.counters(), time=b.time())
        if frames:
            rec['frames'], rec['aux'] = b.frames(), b.aux()
        if ask:
            rec['M'] = b.dynamics()['M']
        out.append(rec)
        b.close()
    for key in out[0]:
        assert np.array_equal(out[0][key], out[1][key]), key
    assert np.abs(out[1]['M']).max() > 1


def test_legacy_verbs_follow_the_reference_restated(oracle_mod):
    P = product()
    for model in ('cassie', 'cassie_tray_box'):
        sim = P.CassieSim(os.path.join(MODELS, model + '.cmodel'))
        u = P.pd_in_t()
        for side, leg in enumerate((u.leftLeg, u.rightLeg)):
            for i in range(5):
                leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
        for _ in range(120):
            sim.step_pd(u)
        q, v = sim.qpos(), sim.qvel()
        want = oracle_dynamics(oracle_mod, model, q, v)
        M = sim.full_mass_matrix()
        assert M.shape == (32, 32) and np.abs(M - want['M'][:32, :32]).max() <= 1e-12 * np.abs(want['M']).max()
        J, err = sim.constraint_jacobian(), sim.constraint_error()
        rows = [3, 4, 5, 9, 10, 11]   # equalities 1 and 3: the achilles-rod connects
        assert J.shape == (6, 32) and err.shape == (6, 1)
        assert np.abs(J - want['J_eq'][rows, :32]).max() <= 1e-12 and np.abs(err[:, 0] - want['eq_err'][rows]).max() <= 1e-12
        Icm = np.array(sim.centroid_inertia()).reshape(3, 3)
        assert np.abs(Icm - want['Icm']).max() <= 1e-10 * np.abs(want['Icm']).max()
        IND = [0, 1, 2, 3, 4, 5, 6, 7, 8, 12, 18, 19, 20, 21, 25, 31]
        import ctypes as C
        buf = (C.c_double * 256)()
        P.lib().cassie_sim_minimal_mass_matrix.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        P.lib().cassie_sim_minimal_mass_matrix(sim.c, buf)
        assert np.abs(np.array(buf[:]).reshape(16, 16) - want['M'][np.ix_(IND, IND)]).max() <= 1e-12 * np.abs(want['M']).max()
        Mp = sim.minimal_mass_matrix()   # the reference wrapper's projection through the constraint Jacobian
        assert Mp.shape == (16, 16) and np.allclose(Mp, Mp.T, atol=1e-9) and np.linalg.eigvalsh(Mp).min() > 0
        Jc = want['J_eq'][rows, :32].copy()
        Jc[:, 0:6] = 0
        dep = [9, 10, 11, 14, 22, 23, 24, 27]
        Jd = Jc[:, IND + dep]
        Jd[Jd < 1e-5] = 0
        G = np.linalg.lstsq(Jd[:, 16:], -Jd[:, :16], rcond=None)[0]
        Pm = np.vstack([np.eye(16), G])
        ref = Pm.T @ want['M'][np.ix_(IND + dep, IND + dep)] @ Pm
        assert np.abs(Mp - ref).max() <= 1e-9 * np.abs(ref).max()
        sim.__del__()


def test_api_behaviour():
    P = product()
    b = P.CassieBatch(8, precision=P.FP64)
    with pytest.raises(RuntimeError):
        b.dynamics()   # before any dynamics launch: -1 with an error
    assert 'dynamics' in P._last_error()
    with pytest.raises(RuntimeError):
        b.torch_view('dyn')
    assert b.row_width('dyn') == P.DYN_WIDTH == 2144
    assert b.neq() == 4
    b.compute_dynamics()
    d = b.dynamics()
    b.sync()
    view = b.torch_view('dyn').cpu().numpy()
    nv = b.nv
    assert np.array_equal(view[:, P.DYN['M']].reshape(8, 40, 40)[:, :nv, :nv], d['M'])
    assert np.array_equal(view[:, P.DYN['bias']][:, :nv], d['bias'])
    assert np.array_equal(view[:, P.DYN['J_eq']].reshape(8, 12, 40)[:, :12, :nv], d['J_eq'])
    assert np.array_equal(view[:, P.DYN['eq_err']], d['eq_err'])
    b.close()


@pytest.mark.parametrize('fp64', [False, True])
def test_large_batch_is_fully_written(fp64):
    """more environments than one round of resident warps: every row is written, and rows of equal states are equal"""
    P = product()
    n = 20000
    b = P.CassieBatch(n, precision=P.FP64 if fp64 else P.FP32)
    b.step(5)
    b.compute_dynamics()
    d = b.dynamics()
    assert np.all(d['M'][:, 0, 0] > 30) and np.all(np.abs(d['bias']).max(axis=1) > 1)
    assert np.array_equal(d['M'][0], d['M'][-1]) and np.array_equal(d['J_eq'][0], d['J_eq'][-1])
    b.close()
