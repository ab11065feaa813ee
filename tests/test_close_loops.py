"""Loop closure (cassie_batch_close_loops) without a GPU: the product's source csrc/loops.inl run in the host emulation (tests/emu/emu_loops.cpp) against
the fp64 oracle's connect rows, on cassie, cassie_mass, cassie_hfield and cassie_tray_box, in both precisions, from three kinds of start states (noise on
the initial state, noise on a settled standing state, per-environment body offsets inside the loops)."""
import numpy as np
import pytest

import loops_support as S

TOL = {False: 1e-12, True: 1e-6}        # the Python defaults of CassieBatch.close_loops
RES = {False: 1e-10, True: 2e-6}        # the oracle's max |p1 - p2| at the result (fp32: the float result evaluated in double)
VRES = {False: 1e-8, True: 1e-4}        # the oracle's max |J qvel| at the result, from qvel ~ N(0, 0.5)
KINDS = ('noisy', 'standing', 'offsets')


def _close(model, fp32, kind, n=16, seed=1, **kw):
    q, v, bp = S.start_states(model, kind, n, seed, fp32)
    e = S.EmuLoops(model, fp32)
    q2, v2, st, k = e.close(q, v, bpos=bp, tol=TOL[fp32], **kw)
    return e, (q, v, bp), (q2, v2, st, k)


def test_free_coordinates_are_the_rod_tarsus_crank_and_plantar_joints():
    t = S.table('cassie')
    qf, vf = S.EmuLoops('cassie', False).free(int(t['nq'][0]), int(t['nv'][0]))
    names = [n for j, n in enumerate(t['names_joint']) if vf[int(t['jnt_dofadr'][j])]]
    assert names == [s + j for s in ('left-', 'right-') for j in ('achilles-rod', 'tarsus', 'foot-crank', 'plantar-rod')]
    assert vf.sum() == 12 and qf.sum() == 14


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', S.MODEL_NAMES)
def test_closes_onto_the_oracles_connect_rows(model, fp32, kind):
    e, (q, v, bp), (q2, v2, st, k) = _close(model, fp32, kind)
    assert k == len(q)
    assert (st[:, 1] >= 1).all(), st[:, 1]
    R = S.OracleRows(model).residuals(q2, v2, bp)
    print(model, fp32, kind, 'iterations', st[:, 1].min(), st[:, 1].max(), 'residual %.2e' % R[:, 0].max(), 'J qvel %.2e' % R[:, 1].max())
    assert R[:, 0].max() <= RES[fp32] and R[:, 1].max() <= VRES[fp32]
    assert np.abs(st[:, 0] - R[:, 0]).max() <= (1e-14 if not fp32 else 5e-7)    # the status row's residual is the oracle's
    assert (st[:, 0] <= TOL[fp32]).all() and (st[:, 3] == 0).all()
    nq, nv = q.shape[1], v.shape[1]
    qf, vf = e.free(nq, nv)
    assert (q2[:, ~qf] == q[:, ~qf]).all() and (v2[:, ~vf] == v[:, ~vf]).all()   # held coordinates bitwise
    t = S.table(model)
    for j in range(int(t['njnt'][0])):
        a = int(t['jnt_qposadr'][j])
        if int(t['jnt_type'][j]) == 1 and qf[a]:
            assert np.abs(np.linalg.norm(q2[:, a:a + 4], axis=1) - 1).max() <= (1e-14 if not fp32 else 3e-7)   # rod quaternions unit


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_unmasked_environments_and_their_status_rows_are_untouched(fp32):
    q, v, bp = S.start_states('cassie', 'noisy', 16, 2, fp32)
    mask = np.arange(16) % 2 == 0
    status = np.full((16, 4), 7.0)
    q2, v2, st, k = S.EmuLoops('cassie', fp32).close(q, v, mask=mask, tol=TOL[fp32], status=status)
    assert k == 8
    assert (q2[~mask] == q[~mask]).all() and (v2[~mask] == v[~mask]).all() and (st[~mask] == 7).all()
    assert (st[mask, 1] >= 1).all() and (q2[mask] != q[mask]).any()


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_a_pose_that_cannot_close_comes_back_unchanged(fp32):
    t = S.table('cassie')
    q, v, _ = S.start_states('cassie', 'noisy', 8, 3, fp32)
    e = S.EmuLoops('cassie', fp32)
    nb = int(t['nbody'][0])
    rods = [list(t['names_body']).index(s + 'achilles-rod') for s in ('left-', 'right-')]
    bp = np.tile(t['body_pos'].reshape(nb, 3), (8, 1, 1))
    bp[:4, rods[0], 2] += 1.0     # a rod's ball a metre from its hip: the 0.5 m rod cannot reach the heel spring
    bp[4:, rods[1], 2] += 1.0
    q2, v2, st, _ = e.close(q, v, bpos=bp, max_iter=50, tol=TOL[fp32])
    assert (st[:, 1] == -1).all() and (q2 == q).all() and (v2 == v).all()
    R = S.OracleRows('cassie').residuals(q, v, bp)
    assert np.abs(st[:, 0] - R[:, 0]).max() <= (1e-14 if not fp32 else 1e-6)   # the residual of the unchanged pose
    big = q.copy()
    big[:, 7:35] += 0.25 * np.random.default_rng(4).standard_normal((8, 28))   # one step from large noise is not enough
    if fp32:
        big = big.astype(np.float32).astype(np.float64)
    q3, v3, st3, _ = e.close(big, v, max_iter=1, tol=TOL[fp32])
    assert (st3[:, 1] == -1).all() and (q3 == big).all() and (v3 == v).all()


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_an_environment_already_closed_keeps_its_qpos_and_has_its_velocity_projected(fp32):
    e, _, (q1, v1, st1, _) = _close('cassie', fp32, 'noisy', n=8)
    v = v1 + 0.3 * np.random.default_rng(5).standard_normal(v1.shape)
    if fp32:
        v = v.astype(np.float32).astype(np.float64)
    q2, v2, st2, _ = e.close(q1, v, tol=TOL[fp32])
    assert (st2[:, 1] == 0).all() and (q2 == q1).all()
    R = S.OracleRows('cassie').residuals(q2, v2)
    assert R[:, 1].max() <= VRES[fp32] and (v2 != v).any()


@pytest.mark.parametrize('kind', KINDS)
@pytest.mark.parametrize('model', S.MODEL_NAMES)
def test_fp64_agrees_with_a_numpy_restatement_on_the_oracles_rows(model, kind):
    e, (q, v, bp), (q2, v2, st, _) = _close(model, False, kind, n=4, seed=6)
    rows = S.OracleRows(model)
    _, vf = e.free(q.shape[1], v.shape[1])
    for i in range(len(q)):
        qn, vn, it = S.restate(model, rows, q[i], v[i], vf, None if bp is None else bp[i], tol=TOL[False], lam=S.LAMBDA[False])
        assert it == st[i, 1]
        assert np.abs(q2[i] - qn).max() <= 1e-9 and np.abs(v2[i] - vn).max() <= 1e-9, (np.abs(q2[i] - qn).max(), np.abs(v2[i] - vn).max())
