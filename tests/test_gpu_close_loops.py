"""GPU: loop closure (cassie_batch_close_loops) through the C-ABI at 4096 environments, half of them selected by a torch mask.  The device equals the host
emulation of the same source (fp64 to 1e-9), its results close onto the fp64 oracle's connect rows, held coordinates and unselected environments keep
their bits, a call captured in a CUDA graph with forward_where equals the eager calls bitwise, compute_dynamics() afterwards shows the equality error
within tol, and every refusal enqueues nothing."""
import ctypes as C

import numpy as np
import pytest

from conftest import product
import loops_support as S

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')

N = 4096
TOL = {False: 1e-12, True: 1e-6}
RES = {False: 1e-10, True: 2e-6}
VRES = {False: 1e-8, True: 1e-4}


@pytest.fixture(scope='module')
def P():
    return product()


def _batch(P, model, fp32, q, v, bp):
    b = P.CassieBatch(N, modelfile=P.model_path(model), precision=P.FP32 if fp32 else P.FP64)
    if bp is not None:
        b.set_env_body_pos(bp)
    b.set_qpos(q)
    b.set_qvel(v)
    return b


def _mask(seed):
    m = np.random.default_rng(seed).permutation(N) < N // 2
    return m, torch.as_tensor(m, device='cuda')


@pytest.mark.parametrize('kind', ('noisy', 'standing', 'offsets'))
@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('model', S.MODEL_NAMES)
def test_device_equals_the_emulation_and_closes_onto_the_oracle(P, model, fp32, kind):
    q, v, bp = S.start_states(model, kind, N, 11, fp32)
    m, mt = _mask(12)
    b = _batch(P, model, fp32, q, v, bp)
    b.close_loops(mt)
    q2, v2, st = b.qpos(), b.qvel(), b.loop_status()
    e = S.EmuLoops(model, fp32)
    qe, ve, se, k = e.close(q, v, mask=m, bpos=bp, tol=TOL[fp32])
    assert k == N // 2
    assert (q2[~m] == q[~m]).all() and (v2[~m] == v[~m]).all() and (st['iterations'][~m] == 0).all() and (st['residual'][~m] == 0).all()
    qf, vf = e.free(q.shape[1], v.shape[1])
    assert (q2[:, ~qf] == q[:, ~qf]).all() and (v2[:, ~vf] == v[:, ~vf]).all()
    assert (st['iterations'][m] >= 1).all(), np.unique(st['iterations'][m])
    if not fp32:
        assert np.abs(q2 - qe).max() <= 1e-9 and np.abs(v2 - ve).max() <= 1e-9
        assert np.abs(st['residual'] - se[:, 0]).max() <= 1e-12 and (st['iterations'] == se[:, 1]).all()
    sel = np.flatnonzero(m)[:128]
    R = S.OracleRows(model).residuals(q2[sel], v2[sel], None if bp is None else bp[sel])
    print(model, fp32, kind, 'iterations', st['iterations'][m].min(), st['iterations'][m].max(), 'residual %.2e' % R[:, 0].max(), 'J qvel %.2e' % R[:, 1].max())
    assert R[:, 0].max() <= RES[fp32] and R[:, 1].max() <= VRES[fp32]
    b.forward_where(mt)
    b.compute_dynamics()
    err = b.dynamics()['eq_err']
    assert np.abs(err[m]).max() <= TOL[fp32] * (1 if not fp32 else 2)   # the step kernel's own fp32 kinematics rounds differently
    b.close()


@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
def test_a_captured_call_equals_the_eager_calls(P, fp32):
    q, v, bp = S.start_states('cassie', 'noisy', N, 13, fp32)
    s = torch.cuda.Stream()
    a, e = (_batch(P, 'cassie', fp32, q, v, None) for _ in range(2))
    a.set_stream(s.cuda_stream)
    mask = torch.zeros(N, dtype=torch.bool, device='cuda')
    a.close_loops(mask)            # the first call allocates the status rows
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        a.close_loops(mask)
        a.forward_where(mask)
    m, mt = _mask(14)
    mask.copy_(mt)
    a.set_qpos(q)
    a.set_qvel(v)
    torch.cuda.synchronize()
    g.replay()
    torch.cuda.synchronize()
    e.close_loops(mt)
    e.forward_where(mt)
    e.sync()
    for f in ('qpos', 'qvel', 'obs'):
        x, y = getattr(a, f)(), getattr(e, f)()
        assert (x == y).all(), f
    sa, se = a.loop_status(), e.loop_status()
    for f in sa:
        assert (sa[f] == se[f]).all(), f
    assert (sa['iterations'][m] >= 1).mean() > 0.99 and (sa['iterations'][~m] == 0).all()   # a rare noisy pose needs more than 20 steps
    del g
    a.close()
    e.close()


def test_refusals_change_nothing(P):
    q, v, _ = S.start_states('cassie', 'noisy', N, 15)
    b = _batch(P, 'cassie', False, q, v, None)
    with pytest.raises(RuntimeError):
        b.loop_status()             # no call yet
    host = np.ones(N, dtype=np.uint8)
    b.L.cassie_batch_close_loops.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double]
    n0 = b.launch_count()
    assert b.L.cassie_batch_close_loops(b.h, host.ctypes.data, 20, 1e-12) == -1      # a host array
    mt = torch.ones(N, dtype=torch.bool, device='cuda')
    for it, tol in ((0, 1e-12), (201, 1e-12), (20, 0.0), (20, -1e-3), (20, float('nan')), (20, float('inf'))):
        with pytest.raises(RuntimeError):
            b.close_loops(mt, max_iter=it, tol=tol)
    assert b.launch_count() == n0 and (b.qpos() == q).all() and (b.qvel() == v).all()
    sim = P.CassieSim(P.model_path('cassie'))
    L = b.L
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    sb = L.cassie_sim_batch(sim.c)
    assert L.cassie_batch_close_loops(C.c_void_p(sb), None, 20, 1e-12) == -1     # the batch of a cassie_sim_t
    assert 'cassie_sim_t' in P._last_error()
    b.close()
