"""GPU: inverse kinematics (cassie_batch_solve_ik) through the C-ABI at 4096 environments, half of them selected by a torch mask.  The device equals the
host emulation of the same source (fp64 to 1e-9), reaches targets posed by the fp64 oracle within the fp32 limits, holds every other coordinate and
every unselected environment bitwise, a graph capture of the target rows being written, solve_ik and forward_where equals the eager calls bitwise, the
frame rows after forward_where match the targets, and every refusal enqueues nothing."""
import ctypes as C

import numpy as np
import pytest

from conftest import product
import ik_support as S
import loops_support as LS

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

N = 4096
REACH = {False: (1e-9, 1e-9), True: (2e-5, 2e-4)}    # position (m), orientation (rad) of the oracle at the result
LOOP = {False: 1e-10, True: 2e-6}


@pytest.fixture(scope='module')
def P():
    return product()


_cases = {}


def _case(model, fp32):
    """N standing starts, targets from N reachable poses (64 distinct, tiled), and the emulation's result for the mask"""
    key = (model, fp32)
    if key not in _cases:
        spec = S.feet(model)
        start, posed = S.reachable(model, 64, 31, fp32=fp32)
        tg = S.target_rows(model, spec, posed)
        if fp32:
            tg = tg.astype(np.float32).astype(np.float64)
        rep = np.arange(N) % 64
        nv = int(LS.table(model)['nv'][0])
        _cases[key] = (spec, start[rep], tg[rep], np.zeros((N, nv)))
    return _cases[key]


def _batch(P, model, fp32, spec, q, v, tg):
    b = P.CassieBatch(N, modelfile=P.model_path(model), precision=P.FP32 if fp32 else P.FP64)
    b.set_qpos(q)
    b.set_qvel(v)
    b.set_ik([s['name'] for s in spec], [s['kind'] for s in spec], [s['frame'] for s in spec], [s['w'] for s in spec])
    b.torch_view('ik_targets').copy_(torch.as_tensor(tg, device='cuda'))
    b.sync()
    return b


def _mask(seed):
    m = np.random.default_rng(seed).permutation(N) < N // 2
    return m, torch.as_tensor(m, device='cuda')


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', S.MODEL_NAMES)
def test_device_equals_the_emulation_and_reaches_the_oracles_targets(P, model, fp32):
    spec, q, tg, v = _case(model, fp32)
    m, mt = _mask(32)
    b = _batch(P, model, fp32, spec, q, v, tg)
    b.solve_ik(mt)
    q2, v2, st = b.qpos(), b.qvel(), b.ik_status()
    assert (q2[~m] == q[~m]).all() and (v2[~m] == v[~m]).all() and (st['outcome'][~m] == 0).all()
    sel = np.flatnonzero(m)[:64]
    qe, ve, se, k = S.EmuIk(model, fp32).solve(q[sel], v[sel], spec, tg[sel])
    assert k == len(sel)
    if not fp32:
        assert np.abs(q2[sel] - qe).max() <= 1e-9 and np.abs(v2[sel] - ve).max() <= 1e-9
        assert (st['outcome'][sel] == se[:, 4]).all() and (st['iterations'][sel] == se[:, 3]).all()
    assert (st['outcome'][m] == 1).all(), np.unique(st['outcome'][m])
    R = S.residuals(model, spec, q2[sel[:32]], tg[sel[:32]])
    print(model, fp32, 'iterations', st['iterations'][m].min(), st['iterations'][m].max(), 'pos %.2e ori %.2e loop %.2e' % tuple(R.max(0)))
    assert R[:, 0].max() <= REACH[fp32][0] and R[:, 1].max() <= REACH[fp32][1] and R[:, 2].max() <= LOOP[fp32]
    dof, _, _, _ = S.EmuIk(model, fp32).columns()
    t = LS.table(model)
    held = np.ones(q.shape[1], dtype=bool)
    for d in dof:
        j = int(t['dof_jntid'][d]) if 'dof_jntid' in t else None
        if j is not None:
            a = int(t['jnt_qposadr'][j])
            held[a:a + (4 if int(t['jnt_type'][j]) == 1 else 1)] = False
    assert (q2[:, held] == q[:, held]).all()
    b.close()


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_a_captured_solve_equals_the_eager_calls_and_the_frames_match(P, fp32):
    spec, q, tg, v = _case('cassie', fp32)
    s = torch.cuda.Stream()
    a, e = (_batch(P, 'cassie', fp32, spec, q, v, tg) for _ in range(2))
    for x in (a, e):
        x.set_frames([sp['name'] for sp in spec], [sp['kind'] for sp in spec])
    a.set_stream(s.cuda_stream)
    mask = torch.zeros(N, dtype=torch.bool, device='cuda')
    src = torch.zeros_like(a.torch_view('ik_targets'))
    view = a.torch_view('ik_targets')
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        view.copy_(src)
        a.solve_ik(mask)
        a.forward_where(mask)
    m, mt = _mask(33)
    mask.copy_(mt)
    src.copy_(torch.as_tensor(tg, device='cuda'))
    a.set_qpos(q)
    a.set_qvel(v)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    e.solve_ik(mt)
    e.forward_where(mt)
    e.sync()
    for f in ('qpos', 'qvel', 'obs', 'frames'):
        x, y = getattr(a, f)(), getattr(e, f)()
        assert (x == y).all(), f
    sa, se = a.ik_status(), e.ik_status()
    for f in sa:
        assert (sa[f] == se[f]).all(), f
    assert (sa['outcome'][m] == 1).all() and (sa['outcome'][~m] == 0).all()
    fr = a.frames()   # [n, nframes, 20]: pos 0..2, quat 3..6 in the world frame; the pelvis is held, so the root targets' world poses are the posed ones
    F = S.OracleFrames('cassie')
    for i in np.flatnonzero(m)[:8]:
        F.set(a.qpos()[i])
        for k, sp in enumerate(spec):
            pw, _ = F._world(sp)
            assert np.abs(fr[i, k, :3] - pw).max() <= (1e-9 if not fp32 else 2e-5)
    del g
    a.close()
    e.close()


def test_refusals_change_nothing(P):
    spec, q, tg, v = _case('cassie', False)
    b = P.CassieBatch(N, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_qpos(q)
    b.set_qvel(v)
    L = b.L
    L.cassie_batch_solve_ik.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_int]
    n0 = b.launch_count()
    assert L.cassie_batch_solve_ik(b.h, None, 100, 1e-10, 0) == -1 and 'no target list' in P._last_error()
    with pytest.raises(RuntimeError, match='no free coordinate'):
        b.set_ik(['cassie-pelvis'], [0])
    b.set_ik([s['name'] for s in spec], [s['kind'] for s in spec], [s['frame'] for s in spec], [s['w'] for s in spec])
    host = np.ones(N, dtype=np.uint8)
    assert L.cassie_batch_solve_ik(b.h, host.ctypes.data, 100, 1e-10, 0) == -1      # a host array
    mt = torch.ones(N, dtype=torch.bool, device='cuda')
    for it, tol in ((0, 1e-10), (501, 1e-10), (100, 0.0), (100, -1.0), (100, float('nan')), (100, float('inf'))):
        with pytest.raises(RuntimeError):
            b.solve_ik(mt, max_iter=it, tol=tol)
    assert b.launch_count() == n0 and (b.qpos() == q).all() and (b.qvel() == v).all()
    sim = P.CassieSim(P.model_path('cassie'))
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    sb = L.cassie_sim_batch(sim.c)
    assert L.cassie_batch_solve_ik(C.c_void_p(sb), None, 100, 1e-10, 0) == -1     # the batch of a cassie_sim_t
    assert 'cassie_sim_t' in P._last_error()
    b.close()
