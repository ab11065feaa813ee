"""Inverse kinematics (cassie_batch_solve_ik) without a GPU: the product's source csrc/ik.inl run in the host emulation (tests/emu/emu_ik.cpp) against the
fp64 oracle's frames (xpos / xquat and the model's sites), Jacobians (cdof) and connect rows (efc), on cassie, cassie_mass, cassie_hfield and
cassie_tray_box (foot bodies where the model has no foot sites), in both precisions."""
import numpy as np
import pytest
from scipy.optimize import least_squares

import ik_support as S
import loops_support as LS

REACH = {False: (1e-9, 1e-9), True: (2e-5, 2e-4)}   # position (m), orientation (rad) of the oracle at the result (fp32: evaluated in double)
LOOP = {False: 1e-10, True: 2e-6}                   # close_loops' limits on the oracle's connect residual


def _held(model, e):
    """qpos entries the solve may not move (every coordinate but the free columns' joints)"""
    t = LS.table(model)
    dof, _, _, _ = e.columns()
    held = np.ones(int(t['nq'][0]), dtype=bool)
    for d in dof:
        j = int(t['dof_jntid'][d]); a = int(t['jnt_qposadr'][j])
        held[a:a + (4 if int(t['jnt_type'][j]) == 1 else 1)] = False
    return held


def test_free_columns_are_the_motors_and_the_loops_joints():
    t = LS.table('cassie')
    dof, lim, lo, hi = S.EmuIk('cassie', False).columns()
    assert len(dof) == 22
    names = sorted({t['names_joint'][int(t['dof_jntid'][d])] for d in dof})
    assert names == sorted(S.MOTOR_JOINTS + [s + j for s in ('left-', 'right-') for j in ('achilles-rod', 'tarsus', 'foot-crank', 'plantar-rod')])


@pytest.mark.parametrize('frame', [S.ROOT, S.WORLD], ids=['root', 'world'])
@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', S.MODEL_NAMES)
def test_reaches_targets_posed_by_the_oracle(model, fp32, frame):
    spec = S.feet(model, frame)
    start, posed = S.reachable(model, 16, 1, fp32=fp32)
    tg = S.target_rows(model, spec, posed)
    if fp32:
        tg = tg.astype(np.float32).astype(np.float64)
    e = S.EmuIk(model, fp32)
    v = np.zeros((16, int(LS.table(model)['nv'][0])))
    q2, v2, st, k = e.solve(start, v, spec, tg)
    assert k == 16 and (st[:, 4] == 1).all(), st[:, 4]
    R = S.residuals(model, spec, q2, tg)
    print(model, fp32, frame, 'iterations', st[:, 3].min(), st[:, 3].max(), 'pos %.2e ori %.2e loop %.2e' % tuple(R.max(0)))
    assert R[:, 0].max() <= REACH[fp32][0] and R[:, 1].max() <= REACH[fp32][1] and R[:, 2].max() <= LOOP[fp32]
    assert np.abs(st[:, 0] - R[:, 0]).max() <= (1e-12 if not fp32 else 5e-6)    # the status row's residuals are the oracle's
    held = _held(model, e)
    assert (q2[:, held] == start[:, held]).all()


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_body_offsets_are_honoured(fp32):
    t = LS.table('cassie')
    spec = S.feet('cassie')
    start, posed = S.reachable('cassie', 8, 2, fp32=fp32)
    nb = int(t['nbody'][0])
    bp = np.tile(t['body_pos'].reshape(nb, 3), (8, 1, 1))
    shin = [list(t['names_body']).index(s + 'shin') for s in ('left-', 'right-')]
    bp[:, shin, 0] += np.random.default_rng(3).uniform(-0.01, 0.01, (8, 2))   # longer / shorter thighs
    if fp32:
        bp = bp.astype(np.float32).astype(np.float64)
    posed_c, _, st0, _ = LS.EmuLoops('cassie', False).close(posed, np.zeros((8, 32)), bpos=bp, max_iter=50, tol=1e-13)
    tg = S.target_rows('cassie', spec, posed_c, bpos=bp)
    q2, _, st, _ = S.EmuIk('cassie', fp32).solve(start, np.zeros((8, 32)), spec, tg, bpos=bp)
    assert (st[:, 4] == 1).all()
    R = S.residuals('cassie', spec, q2, tg, bp)
    assert R[:, 0].max() <= REACH[fp32][0] and R[:, 1].max() <= REACH[fp32][1] and R[:, 2].max() <= LOOP[fp32]


def _unreachable(model, n, seed):
    """targets out of reach (a foot 0.6-0.8 m too low) or past a hip range (a foot 0.4-0.5 m further out or in, beyond the hip roll's range)"""
    spec = S.feet(model)
    start, posed = S.reachable(model, n, seed)
    tg = S.target_rows(model, spec, posed)
    rng = np.random.default_rng(seed)
    half = n // 2
    tg[:half, 0, 2] -= rng.uniform(0.6, 0.8, half)
    side = np.where(np.arange(n - half) % 2 == 0, 1.0, -1.0)
    tg[half:, 0, 1] += side * rng.uniform(0.4, 0.5, n - half)
    return spec, start, tg


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_unreachable_targets_give_the_best_effort_within_range(model, fp32):
    spec, start, tg = _unreachable(model, 8, 5)
    if fp32:
        tg = tg.astype(np.float32).astype(np.float64)
    e = S.EmuIk(model, fp32)
    nv = int(LS.table(model)['nv'][0])
    q2, _, st, _ = e.solve(start, np.zeros((8, nv)), spec, tg, max_iter=300)
    assert (st[:, 4] == 2).all(), st[:, 4]
    R = S.residuals(model, spec, q2, tg)
    assert R[:, 2].max() <= LOOP[fp32]                                           # the loops are closed
    mq, mr = S.motor_qpos(model), S.motor_range(model)
    if fp32:
        mr = mr.astype(np.float32).astype(np.float64)                              # the range in the batch precision
    assert ((q2[:, mq] >= mr[:, 0]) & (q2[:, mq] <= mr[:, 1])).all()           # every motor inside its range, bitwise
    F = S.OracleFrames(model)
    for i in range(8):
        F.set(q2[i]); f2 = S.objective(F, spec, tg[i])
        F.set(start[i]); f0 = S.objective(F, spec, tg[i])
        assert f2 <= f0 * (1 + 1e-12)                                              # no larger than at the (closed) start
    assert (st[:, 7] >= 1).any()                                                  # some are held by a range


def test_unreachable_results_are_first_order_optimal_on_the_oracles_jacobians():
    model = 'cassie'
    spec, start, tg = _unreachable(model, 8, 6)
    e = S.EmuIk(model, False)
    q2, _, st, _ = e.solve(start, np.zeros((8, 32)), spec, tg, max_iter=400)
    assert (st[:, 4] == 2).all()
    dof, lim, lo, hi = e.columns()
    t = LS.table(model)
    qa = np.array([int(t['jnt_qposadr'][int(t['dof_jntid'][d])]) for d in dof])
    F = S.OracleFrames(model)
    worst = 0.0
    for i in range(8):
        F.set(q2[i])
        g = S.gradient(F, spec, tg[i])[dof]
        _, Jc = F.connect()
        Jc = Jc[:, dof]
        x = q2[i, qa]
        at_lo, at_hi = lim & (x <= lo), lim & (x >= hi)
        off = ~(at_lo | at_hi)
        mu = np.linalg.lstsq(Jc[:, off].T, -g[off], rcond=1e-10)[0]                 # the connect rows' multipliers on the columns off their bounds
        pg = g + Jc.T @ mu
        worst = max(worst, np.abs(pg[off]).max())
        assert (pg[at_lo] >= -1e-8).all() and (pg[at_hi] <= 1e-8).all(), (pg[at_lo], pg[at_hi])   # descent points out of the range
    print('projected gradient %.2e' % worst)
    assert worst <= 5e-8   # the steps stop once a step no longer lowers the residual in double: 2.4e-8 at worst here


def test_out_of_reach_results_are_no_worse_than_scipys_bounded_least_squares():
    # the targets below reach (the first half of _unreachable's); past a hip range the residual has several local minima on the range's faces, and from
    # the same start the solve and scipy may stop in different ones
    model = 'cassie'
    spec, start, tg = _unreachable(model, 8, 7)
    start, tg = start[:4], tg[:4]
    q2, _, st, _ = S.EmuIk(model, False).solve(start, np.zeros((4, 32)), spec, tg, max_iter=400)
    mq, mr = S.motor_qpos(model), S.motor_range(model)
    loops = LS.EmuLoops(model, False)
    F = S.OracleFrames(model)

    def rows(m, i):
        q = start[i].copy(); q[mq] = m
        qc, _, s, _ = loops.close(q[None], np.zeros((1, 32)), max_iter=50, tol=1e-13)
        F.set(qc[0])
        out = []
        for k, sp in enumerate(spec):
            dpos, ev = F.rows(sp, tg[i, k])
            out.append(np.asarray(sp['w'][:3]) * dpos); out.append(np.asarray(sp['w'][3:]) * ev)
        return np.concatenate(out)

    for i in range(4):
        r = least_squares(rows, start[i, mq], bounds=(mr[:, 0], mr[:, 1]), args=(i,), xtol=1e-12, ftol=1e-12, gtol=1e-12)
        F.set(q2[i])
        mine = np.sqrt(S.objective(F, spec, tg[i]))
        print(i, 'ik %.6e scipy %.6e' % (mine, np.linalg.norm(r.fun)))
        assert mine <= np.linalg.norm(r.fun) + 1e-6


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_velocities_are_fitted_to_the_target_rows(fp32):
    model = 'cassie'
    spec = S.feet(model)
    start, posed = S.reachable(model, 8, 8)
    rng = np.random.default_rng(8)
    v = np.zeros((8, 32)); v[:, :32] = 0.5 * rng.standard_normal((8, 32))
    _, vc, _, _ = LS.EmuLoops(model, False).close(posed, v, max_iter=50, tol=1e-13)   # a loop-consistent (q, qvel)
    tg = S.target_rows(model, spec, posed, vc)
    if fp32:
        tg = tg.astype(np.float32).astype(np.float64)
    start = start.copy(); start[:, :7] = posed[:, :7]
    v0 = vc.copy(); v0[:, 6:] = 0                                                # the pelvis motion held, the rest to be fitted
    if fp32:
        start, v0 = start.astype(np.float32).astype(np.float64), v0.astype(np.float32).astype(np.float64)
    e = S.EmuIk(model, fp32)
    q2, v2, st, _ = e.solve(start, v0, spec, tg, velocities=1)
    assert (st[:, 4] == 1).all()
    F = S.OracleFrames(model)
    worst, jq = 0.0, 0.0
    for i in range(8):
        F.set(q2[i], v2[i])
        for k, sp in enumerate(spec):
            lv, av = F.velocity(sp, v2[i])
            tq = tg[i, k, 3:7] / np.linalg.norm(tg[i, k, 3:7])
            w = np.asarray(sp['w'])
            err = np.concatenate([(lv - tg[i, k, 7:10])[w[:3] != 0], (S._q2m(tq).T @ (av - tg[i, k, 10:13]))[w[3:] != 0]])
            worst = max(worst, np.abs(err).max())
        _, Jc = F.connect()
        jq = max(jq, np.abs(Jc @ v2[i]).max())
    print('velocity error %.2e J_eq qvel %.2e' % (worst, jq))
    assert worst <= (1e-9 if not fp32 else 1e-4) and jq <= (1e-8 if not fp32 else 1e-4)
    assert (v2[:, :6] == v0[:, :6]).all()
    q3, v3, st3, _ = e.solve(start, v0, spec, tg, velocities=0)
    mv = [int(LS.table(model)['jnt_dofadr'][list(LS.table(model)['names_joint']).index(j)]) for j in S.MOTOR_JOINTS]
    assert (v3[:, mv] == v0[:, mv]).all() and (st3[:, 6] == 0).all()            # the motors keep their qvel bitwise


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_masked_environments_and_a_pose_at_its_targets_keep_their_bits(fp32):
    spec = S.feet('cassie')
    start, posed = S.reachable('cassie', 16, 9, fp32=fp32)
    tg = S.target_rows('cassie', spec, posed)
    e = S.EmuIk('cassie', fp32)
    mask = np.arange(16) % 2 == 0
    status = np.full((16, S.IK_SLOT), 7.0)
    v = np.zeros((16, 32))
    q2, v2, st, k = e.solve(start, v, spec, tg, mask=mask, status=status)
    assert k == 8 and (q2[~mask] == start[~mask]).all() and (v2[~mask] == v[~mask]).all() and (st[~mask] == 7).all()
    assert (st[mask, 4] == 1).all()
    q3, _, st3, _ = e.solve(q2[mask], v[mask], spec, S.target_rows('cassie', spec, q2[mask]))   # the pose is at its (own) targets
    assert (st3[:, 4] == 1).all() and (st3[:, 3] == 0).all() and (q3 == q2[mask]).all()


def test_an_open_start_that_cannot_close_is_kept():
    t = LS.table('cassie')
    spec = S.feet('cassie')
    start, posed = S.reachable('cassie', 4, 10)
    tg = S.target_rows('cassie', spec, posed)
    nb = int(t['nbody'][0])
    bp = np.tile(t['body_pos'].reshape(nb, 3), (4, 1, 1))
    rod = list(t['names_body']).index('left-achilles-rod')
    bp[:, rod, 2] += 1.0     # the rod's ball a metre from its hip: the loop cannot close
    q2, v2, st, _ = S.EmuIk('cassie', False).solve(start, np.zeros((4, 32)), spec, tg, bpos=bp)
    assert (st[:, 4] == -1).all() and (q2 == start).all()


def test_refused_target_lists():
    e = S.EmuIk('cassie', False)
    t = LS.table('cassie')
    pelvis = dict(S.feet('cassie')[0], body=list(t['names_body']).index('cassie-pelvis'), kind=0, pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]))
    q = LS.standing('cassie')[None]
    assert e.solve(q, np.zeros((1, 32)), [pelvis], np.zeros((1, 4, 16)))[3] == -1   # nothing free moves the pelvis
    tb = S.EmuIk('cassie_tray_box', False)
    tt = LS.table('cassie_tray_box')
    box = dict(pelvis, body=int(tt['nbody'][0]) - 1)
    q = LS.standing('cassie_tray_box')[None]
    assert tb.solve(q, np.zeros((1, int(tt['nv'][0]))), [box], np.zeros((1, 4, 16)))[3] == -1   # nor the extra free body
