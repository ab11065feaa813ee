"""GPU: inverse rows (cassie_batch_inverse, launch mode 6) -- the F_FR kernel instances against the fp64 oracle's restatement of mj_inverse
(tests/inverse_support.py) per sampled environment, with per-environment rows, the zero-copy round trip from the acceleration rows, bitwise neutrality for
stepping and the API's behaviour.  CPU twins (host emulation): tests/test_inverse.py."""
import numpy as np
import pytest

from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product
from contact_support import random_contact
from inverse_support import inverse, oracle_at, scale
from mechanics_support import random_mechanics
from test_env_body_pos import offsets
from test_hfield import terrain
from test_inverse import FP32_BARS, gait_row

pytestmark = pytest.mark.gpu


def _batch(model, fp64, n, hf=None):
    P = product()
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64 if fp64 else P.FP32)
    if hf is not None:
        b.set_hfield_data(hf)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    b.forward()
    return P, b


def _checkpoints(P, b):
    """the batch through a stance, a gait (targets swung every 25 ticks) and a fall with the motors off; yields the phase at two points of each"""
    n = b.n
    for ph in ('stance', 'gait', 'fall'):
        for k in range(2):
            for c in range(4):
                if ph == 'gait':
                    r = gait_row(300 + 100 * k + 25 * c)
                    b.set_pd(P.pd_rows(n, pTarget=r[10:20], pGain=PD_PGAIN, dGain=PD_DGAIN))
                elif ph == 'fall':
                    b.set_pd(P.pd_rows(n))
                b.step(25)
            yield ph


def _parity(O, model, fp64, n, nsample):
    """errors of nsample sampled environments against the restatement, per sample relative to inverse_support.scale, at six checkpoints and three
    qacc each (the oracle's solved qacc, zero, the solved one perturbed); samples whose row or contact count differs from the oracle's are counted apart"""
    hf = terrain(7) if model == 'cassie_hfield' else None
    P, b = _batch(model, fp64, n, hf)
    rng = np.random.default_rng(5)
    sample = rng.choice(n, nsample, replace=False) if nsample < n else np.arange(n)
    err = dict(qfrc_inverse=[], qfrc_constraint=[])
    counts_equal, active, mismatched = True, 0, 0
    for ph in _checkpoints(P, b):
        q, v = b.qpos(), b.qvel()
        os_ = {e: oracle_at(O, model, q[e], v[e], hfield=hf) for e in sample}
        solved = np.zeros((n, b.nv))
        for e, o in os_.items():
            solved[e] = o.arr('qacc')
        for kind, qa in (('solved', solved), ('zero', np.zeros((n, b.nv))), ('perturbed', solved + rng.normal(0, 1, solved.shape) * (1 + np.abs(solved)) * 0.3)):
            b.compute_inverse(qa)
            got = b.inverse()
            for e, o in os_.items():
                want = inverse(o, model, qa[e])
                same = (got['nefc'][e], got['ncon'][e]) == (want['nefc'], want['ncon'])
                counts_equal = counts_equal and same
                if not same:   # a contact the other precision does not make: compared only for its count
                    mismatched += 1
                    continue
                for key in err:
                    err[key].append(np.abs(got[key][e] - want[key]).max() / scale(want))
                active += int((want['f'][want['ineq']] > 0).sum())
        for o in os_.values():
            o.close()
    b.close()
    return {k: np.array(x) for k, x in err.items()}, counts_equal, active, mismatched


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box', 'cassie_hfield'])
def test_fp64_inverse_follows_the_oracle(oracle_mod, model):
    err, counts_equal, active, _ = _parity(oracle_mod, model, True, 256, 32)
    print(model, {k: (x.max(), np.median(x)) for k, x in err.items()}, active)
    assert counts_equal and active > 0
    assert err['qfrc_inverse'].max() <= 1e-9 and err['qfrc_constraint'].max() <= 1e-9, err


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_fp64_inverse_with_per_environment_rows(oracle_mod, model):
    """four environments with their own mechanics, body offsets and contact softness against four oracles given the same tables"""
    n = 4
    mech = [np.stack(x) for x in zip(*[random_mechanics(model, 20 + e) for e in range(n)])]
    bp = np.stack([offsets(model, 20 + e) for e in range(n)])
    ct = [np.stack(x) for x in zip(*[random_contact(model, 20 + e) for e in range(n)])]
    P, b = _batch(model, True, n)
    b.set_env_mechanics(*mech)
    b.set_env_body_pos(bp)
    b.set_env_contact(*ct)
    worst, counts_equal = 0.0, True
    rng = np.random.default_rng(3)
    for ph in _checkpoints(P, b):
        q, v = b.qpos(), b.qvel()
        os_ = [oracle_at(oracle_mod, model, q[e], v[e], inertia=mech[0][e], armature=mech[1][e], stiffness=mech[2][e], springref=mech[3][e],
                         body_pos=bp[e], geom_solref=ct[0][e], geom_solimp=ct[1][e], geom_solmix=ct[2][e]) for e in range(n)]
        qa = np.stack([o.arr('qacc').copy() for o in os_]) + rng.normal(0, 1, (n, b.nv))
        b.compute_inverse(qa)
        got = b.inverse()
        for e, o in enumerate(os_):
            want = inverse(o, model, qa[e])
            counts_equal = counts_equal and (got['nefc'][e], got['ncon'][e]) == (want['nefc'], want['ncon'])
            worst = max(worst, np.abs(got['qfrc_inverse'][e] - want['qfrc_inverse']).max() / scale(want))
            o.close()
    b.close()
    print(model, worst)
    assert counts_equal and worst <= 1e-9, worst


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_fp32_inverse_4096_sampled(oracle_mod, model):
    """fp32 states against the fp64 oracle at the same qpos / qvel: a contact at distance ~0 can be made in one precision and not in the other (measured
    on an H100: at one gait checkpoint of cassie_tray_box the cup touches the tray in fp32 only, 192 of 1152 samples, all of them at that checkpoint);
    those samples are compared by their counts only, the rest against the emulation's bars"""
    err, counts_equal, active, mismatched = _parity(oracle_mod, model, False, 4096, 64)
    print(model, {k: (x.max(), np.percentile(x, 90), np.median(x)) for k, x in err.items()}, 'count mismatches', mismatched)
    assert mismatched <= 0.25 * (len(err['qfrc_inverse']) + mismatched), mismatched
    for key, bar in FP32_BARS.items():
        assert err[key].max() <= bar, (key, err[key].max())


def test_zero_copy_round_trip_from_the_acceleration_rows(oracle_mod):
    """forward() with acceleration rows; their qacc copied into torch_view('inv_qacc') on the batch's stream; compute_inverse(None) equals the oracle's
    inverse at the same state and qacc, and the device rows equal what inverse() copies"""
    import torch
    P, b = _batch('cassie', True, 64)
    b.set_stream(torch.cuda.current_stream().cuda_stream)
    b.enable_accelerations()
    b.step(300)
    b.forward()
    iq, acc = b.torch_view('inv_qacc'), b.torch_view('acc')
    iq[:, :b.nv].copy_(acc[:, P.ACC['qacc']][:, :b.nv])
    b.compute_inverse(None)
    got, qa, q, v = b.inverse(), b.qacc(), b.qpos(), b.qvel()
    view = b.torch_view('inv').cpu().numpy()
    assert np.array_equal(view[:, P.INV['qfrc_inverse']][:, :b.nv], got['qfrc_inverse'])
    for e in range(0, 64, 8):
        o = oracle_at(oracle_mod, 'cassie', q[e], v[e])
        want = inverse(o, 'cassie', qa[e])
        assert np.abs(got['qfrc_inverse'][e] - want['qfrc_inverse']).max() <= 1e-9 * scale(want), e
        o.close()
    b.close()


def test_inverse_launches_leave_stepping_bitwise_alone():
    """an inverse launch every 10 ticks: qpos, qvel, obs, aux, frames, acceleration rows and counters bitwise those of a twin that never asked"""
    P = product()
    n = 128
    twins = []
    for _ in range(2):
        b = P.CassieBatch(n, modelfile=P.model_path('cassie_tray_box'), precision=P.FP64)
        b.enable_aux()
        b.set_frames(['left-foot', 'right-foot', 'cassie-pelvis'])
        b.enable_accelerations()
        b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        twins.append(b)
    a, b = twins
    rng = np.random.default_rng(9)

    def rows(x):
        return dict(qpos=x.qpos(), qvel=x.qvel(), obs=x.obs(), aux=x.aux(), frames=x.frames(), qacc=x.qacc(), counters=x.counters(),
                    cacc=x.body_accelerations())
    for k in range(300):
        if k == 150:
            a.set_pd(P.pd_rows(n))
            b.set_pd(P.pd_rows(n))
        a.step(1)
        b.step(1)
        if k % 10 == 0:
            before = rows(b)
            b.compute_inverse(rng.normal(0, 5, (n, b.nv)))
            b.inverse()
            after = rows(b)
            for key in before:
                assert np.array_equal(before[key], after[key]), (k, key)
    ra, rb = rows(a), rows(b)
    for key in ra:
        assert np.array_equal(ra[key], rb[key]), key
    a.close()
    b.close()


def test_api():
    P = product()
    b = P.CassieBatch(8, precision=P.FP32)
    with pytest.raises(RuntimeError):
        b.inverse()                  # no launch yet
    with pytest.raises(RuntimeError):
        b.compute_inverse(None)      # no input rows yet
    assert tuple(b.torch_view('inv_qacc').shape) == (8, 32) and tuple(b.torch_view('inv').shape) == (8, P.INV_WIDTH)
    assert float(b.torch_view('inv_qacc').abs().max()) == 0   # allocated zeroed
    b.compute_inverse(None)          # the rows exist now: qacc = 0
    out = b.inverse()
    assert out['qfrc_inverse'].shape == (8, 32) and out['nefc'].shape == (8,) and (out['dropped'] == 0).all()
    b.step(200)
    b.compute_inverse(np.zeros((8, 32)))
    out = b.inverse()
    assert (out['ncon'] >= 1).all() and (out['nefc'] >= 12).all()
    b.close()
