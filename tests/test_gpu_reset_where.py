"""GPU: device-side resets (cassie_batch_set_reset_bank / reset_where / forward_where).  A restore from the bank equals, bitwise, the snapshot rows of
the chosen entry, and what follows it equals the trajectory that entry's environment had; reset_where from a bank of the initial state equals the host
verb cassie_batch_reset(mask); forward_where equals a whole-batch forward for the masked environments; a captured CUDA graph equals the eager calls;
and every refusal leaves the batch as it was."""
import ctypes as C

import numpy as np
import pytest

from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_frames import all_frames

pytestmark = pytest.mark.gpu
torch = pytest.importorskip('torch')


@pytest.fixture(scope='module')
def P():
    return product()


def _pd(P, n, seed):
    rng = np.random.default_rng(seed)
    t = np.asarray(PD_TARGET)[None, :] + rng.uniform(-0.05, 0.05, (n, 10))
    return P.pd_rows(n, pTarget=t, pGain=PD_PGAIN, dGain=PD_DGAIN)


def _batch(P, model, fp64, n, est=True, aux=True, applied=True, frames=8, acc=True, seed=0, frame_offset=0):
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=P.FP64 if fp64 else P.FP32)
    if est:
        b.enable_estimator_device(True)
    else:
        b.enable_estimator_device(False)
    if aux:
        b.enable_aux()
    if frames:
        names, kinds = all_frames(model)
        b.set_frames(names[frame_offset:frame_offset + frames], kinds[frame_offset:frame_offset + frames])
    if acc:
        b.enable_accelerations()
    if applied:
        rng = np.random.default_rng(seed + 1)
        nb = b.L.cassie_batch_nbody(b.h)
        x = np.zeros((n, nb, 6))
        x[:, 1, :3] = rng.uniform(-20, 20, (n, 3))
        b.set_applied_forces(x, rng.uniform(-1, 1, (n, b.nv)))
    b.set_pd(_pd(P, n, seed))
    b.reset()
    return b


def _raw(b, field, width):
    ptr = b.device_ptr(field)
    assert ptr

    class _A:
        pass
    a = _A()
    a.__cuda_array_interface__ = dict(shape=(b.n, width), typestr='<f4' if b.precision == 0 else '<f8', data=(ptr, False), version=2)
    return torch.as_tensor(a, device='cuda').cpu().numpy().copy()


def _state(b):
    """every row a restore writes, as the caller reads them: torch views, the estimator's outputs and the controller-stage state"""
    b.sync()
    s = dict(qpos=b.torch_view('qpos').cpu().numpy().copy(), qvel=b.torch_view('qvel').cpu().numpy().copy(), obs=b.torch_view('obs').cpu().numpy().copy(),
             xfrc=b.torch_view('xfrc').cpu().numpy().copy(), cst=_raw(b, 'cst', 192), qacc_ws=_raw(b, 'qacc_ws', b.row_width('qvel')), time=b.time())
    for f in ('aux', 'frames', 'acc', 'applied'):
        if b.device_ptr(f) and b.row_width(f) > 0:
            s[f] = b.torch_view(f).cpu().numpy().copy()
    for k, v in b.actuator_state().items():
        s['act_' + k] = v
    try:
        s['est'] = b.estimator()
    except RuntimeError:
        pass
    return s


def _same(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _masks(n, k, seed, frac=0.1):
    rng = np.random.default_rng(seed)
    m = rng.random(n) < frac
    m[:2] = True
    ent = rng.integers(-3 * k, 3 * k, n).astype(np.int32)
    ent[0], ent[1] = -1, k + 3
    return m, ent, (ent.view(np.uint32) % np.uint32(k)).astype(np.int64)


def _reset(b, m, ent):
    mt, et = torch.as_tensor(m, device='cuda'), torch.as_tensor(ent, device='cuda')
    torch.cuda.synchronize()
    b.reset_where(mt, et)
    b.sync()


CASES = [('cassie', False, 4096), ('cassie', True, 64), ('cassie_tray_box', False, 256)]


@pytest.mark.parametrize('model,fp64,n', CASES)
def test_bitwise_restore_and_continuation(P, model, fp64, n):
    b = _batch(P, model, fp64, n, seed=3)
    b.step(300)
    S = b.get_state()
    rows_S = _state(b)
    K = 64
    envs = np.random.default_rng(5).choice(n, K, replace=n < K)
    b.set_reset_bank(S, envs)
    assert b.reset_bank_size() == K
    b.step(200)
    pre = _state(b)
    m, ent, j = _masks(n, K, 9)
    _reset(b, m, ent)
    post = _state(b)
    src = envs[j]
    for f in post:
        assert _same(post[f][m], rows_S[f][src[m]]), f
        assert _same(post[f][~m], pre[f][~m]), f
    # continuation: a restored environment follows the trajectory its bank entry's environment had from S (a second batch restored from S, with the PD
    # rows permuted to match)
    pdS = _pd(P, n, 3)
    pdA = pdS.copy()
    pdA[m] = pdS[src[m]]
    b.set_pd(pdA)
    t = _batch(P, model, fp64, n, seed=3)
    t.set_state(S)
    t.set_pd(pdS)
    b.step(100)
    t.step(100)
    ra, rt = _state(b), _state(t)
    for f in ra:
        assert _same(ra[f][m], rt[f][src[m]]), f
    b.free_state(S)
    b.close()
    t.close()


@pytest.mark.parametrize('model,fp64,n', [('cassie', False, 1024), ('cassie', True, 64)])
def test_bank_lacking_est_and_applied_rows_zeroes_them(P, model, fp64, n):
    """the helper batch has no estimator and no applied-force rows: the restored environments' applied rows read zero and their filters start afresh,
    exactly as in a batch restored from that snapshot by set_state"""
    h = _batch(P, model, fp64, 32, est=False, applied=False, seed=4)
    h.step(150)
    S0 = h.get_state()
    b = _batch(P, model, fp64, n, seed=6)
    b.step(120)
    b.set_reset_bank(S0, k=32)
    pre = _state(b)
    m, ent, j = _masks(n, 32, 10)
    _reset(b, m, ent)
    post = _state(b)
    assert not post['applied'][m].any()
    rows_S0 = _state(h)
    for f in ('qpos', 'qvel', 'qacc_ws', 'cst', 'obs', 'aux', 'frames', 'acc', 'time'):
        assert _same(post[f][m], rows_S0[f][j[m]]), f
    for f in post:
        assert _same(post[f][~m], pre[f][~m]), f
    # the filters start afresh: the same as set_state of S0 into a batch with estimator and applied rows, 50 ticks on
    t = _batch(P, model, fp64, 32, seed=6)
    t.set_state(S0)
    pd = _pd(P, n, 6)
    pdt = np.repeat(pd[:1], 32, 0)
    pd[m] = pd[0]
    b.set_pd(pd)
    t.set_pd(pdt)
    b.step(50)
    t.step(50)
    ra, rt = _state(b), _state(t)
    for f in ra:
        assert _same(ra[f][m], rt[f][j[m]]), f
    for x in (h, b, t):
        x.close()


def test_other_frame_list_leaves_frames_alone(P):
    n = 512
    h = _batch(P, 'cassie', False, 16, seed=7, frame_offset=1)
    h.step(100)
    S = h.get_state()
    b = _batch(P, 'cassie', False, n, seed=8)
    b.step(100)
    b.set_reset_bank(S, k=16)
    pre = _state(b)
    m, ent, j = _masks(n, 16, 11)
    _reset(b, m, ent)
    post, rows_S = _state(b), _state(h)
    assert _same(post['frames'], pre['frames']) and _same(post['acc'], pre['acc'])
    for f in ('qpos', 'qvel', 'cst', 'obs', 'aux', 'applied', 'est'):
        assert _same(post[f][m], rows_S[f][j[m]]), f
    h.close()
    b.close()


@pytest.mark.parametrize('fp64,n', [(False, 4096), (True, 64)])
def test_equals_the_host_reset(P, fp64, n):
    """a bank of the state right after cassie_batch_reset(NULL), entry 0 for everyone: the same rows as cassie_batch_reset(mask) on a twin"""
    a, t = (_batch(P, 'cassie', fp64, n, est=False, aux=False, frames=0, acc=False, seed=12) for _ in range(2))
    S = a.get_state()
    a.set_reset_bank(S, envs=[0])
    qfrc = np.tile(np.random.default_rng(13).uniform(-1, 1, a.nv), (n, 1))
    for x in (a, t):
        x.set_applied_forces(qfrc=qfrc)
        x.step(150)
    m = np.random.default_rng(14).random(n) < 0.1
    torch.cuda.synchronize()
    a.reset_where(torch.as_tensor(m, device='cuda'), torch.zeros(n, dtype=torch.int32, device='cuda'))
    t.reset(m.astype(np.uint8))
    ra, rt = _state(a), _state(t)
    for f in ('qpos', 'qvel', 'qacc_ws', 'cst', 'xfrc', 'applied', 'act_torque_delay', 'act_drive_filter', 'act_joint_x', 'act_joint_y'):
        assert _same(ra[f], rt[f]), f
    a.step(50)
    t.step(50)
    ra, rt = _state(a), _state(t)
    for f in ra:
        assert _same(ra[f], rt[f]), f
    a.close()
    t.close()


def test_forward_where_equals_a_whole_batch_forward(P):
    n = 256
    b = _batch(P, 'cassie', False, n, est=False, frames=0, acc=False, seed=15)
    pos = b.env_body_pos()
    pos[3, 2, 2] += 0.003   # environment 3 has its own body offsets: the forward must use them
    b.set_env_body_pos(pos)
    b.step(100)
    S = b.get_state()
    b.set_reset_bank(S, k=n)
    b.step(50)
    m, ent, _ = _masks(n, n, 16)
    m[3] = True
    _reset(b, m, ent)
    q = b.torch_view('qpos')
    noise = torch.as_tensor(np.random.default_rng(17).uniform(-0.01, 0.01, (n, 28)) * m[:, None], device='cuda', dtype=q.dtype)
    q[:, 7:35] += noise
    torch.cuda.synchronize()
    S2 = b.get_state()
    pre = _state(b)
    mt = torch.as_tensor(m, device='cuda')
    torch.cuda.synchronize()
    b.forward_where(mt)
    x = _state(b)
    b.set_state(S2)
    b.forward()
    y = _state(b)
    for f in ('qpos', 'qvel', 'qacc_ws', 'cst', 'obs', 'aux', 'applied'):
        assert _same(x[f][m], y[f][m]), f
        assert _same(x[f][~m], pre[f][~m]), f
    assert not _same(x['cst'][3], pre['cst'][3]) and not _same(x['aux'][3], pre['aux'][3])   # the noisy pose's sensor data and derived quantities
    b.close()


def test_graph_capture_equals_the_eager_calls(P):
    n = 512
    s = torch.cuda.Stream()
    a, e = (_batch(P, 'cassie', False, n, est=False, frames=0, acc=False, seed=18) for _ in range(2))
    a.set_stream(s.cuda_stream)
    for x in (a, e):
        x.step(100)
        x.set_reset_bank(x.get_state(), k=n)
        x.step(30)
    mask = torch.zeros(n, dtype=torch.bool, device='cuda')
    entry = torch.zeros(n, dtype=torch.int32, device='cuda')
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        a.reset_where(mask, entry)
        a.forward_where(mask)
    for seed in (19, 20):
        m, ent, _ = _masks(n, n, seed, frac=0.3)
        mask.copy_(torch.as_tensor(m))
        entry.copy_(torch.as_tensor(ent))
        torch.cuda.synchronize()
        g.replay()
        mt, et = torch.as_tensor(m, device='cuda'), torch.as_tensor(ent, device='cuda')
        torch.cuda.synchronize()
        e.reset_where(mt, et)
        e.forward_where(mt)
        torch.cuda.synchronize()
        ra, re_ = _state(a), _state(e)
        for f in ra:
            assert _same(ra[f], re_[f]), f
        for x in (a, e):
            x.step(20)
    del g
    a.close()
    e.close()


def test_refusals_change_nothing(P):
    n = 64
    L = P.lib()
    b = _batch(P, 'cassie', False, n, est=False, frames=0, acc=False, seed=21)
    m = torch.ones(n, dtype=torch.bool, device='cuda')
    b.step(10)
    before = _state(b)

    def refused(fn, *words):
        with pytest.raises(RuntimeError) as ei:
            fn()
        for w in words:
            assert w in str(ei.value), (w, str(ei.value))

    refused(lambda: b.reset_where(m), 'no reset bank')
    S = b.get_state()
    b.set_reset_bank(S, k=n)
    host = np.ones(n, np.uint8)
    assert L.cassie_batch_reset_where(b.h, C.c_void_p(host.ctypes.data), None) == -1
    assert 'device or managed memory' in P._last_error()
    assert L.cassie_batch_forward_where(b.h, C.c_void_p(host.ctypes.data)) == -1
    assert L.cassie_batch_reset_where(b.h, None, None) == -1
    b.enable_estimator(forces=True, filters=True)
    refused(lambda: b.reset_where(m), 'estimator')
    b.enable_estimator(forces=False, filters=False)
    d = P.CassieBatch(8, precision=P.FP64)
    Sd = d.get_state()
    refused(lambda: b.set_reset_bank(Sd, k=8), 'precision')
    refused(lambda: b.set_reset_bank(S, envs=[0, n]), 'outside')
    refused(lambda: b.set_reset_bank(S, envs=[-1]), 'outside')
    assert b.reset_bank_size() == n   # the old bank is kept
    for f, v in _state(b).items():
        assert _same(v, before[f]), f
    # applied-force rows without contact rows yet: the first extended launch would allocate them
    c = P.CassieBatch(n)
    c.enable_aux()
    c.enable_applied_forces(True)
    ones = torch.ones(n, dtype=torch.bool, device='cuda')
    torch.cuda.synchronize()
    refused(lambda: c.forward_where(ones), 'cassie_batch_forward')
    c.forward()
    c.forward_where(ones)
    c.sync()
    # the batch of a legacy simulator
    sim = P.CassieSim(P.model_path('cassie'))
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    L.cassie_batch_state_free.argtypes = [C.c_void_p, C.c_void_p]
    sb = L.cassie_sim_batch(sim.c)
    Ss = L.cassie_batch_state_alloc(sb)
    assert L.cassie_batch_get_state(sb, C.c_void_p(Ss)) == 0
    assert L.cassie_batch_set_reset_bank(sb, C.c_void_p(Ss), None, 1) == 0
    one = torch.ones(1, dtype=torch.uint8, device='cuda')
    assert L.cassie_batch_reset_where(sb, C.c_void_p(one.data_ptr()), None) == -1
    assert 'cassie_sim_t' in P._last_error()
    L.cassie_batch_set_reset_bank(sb, None, None, 0)
    L.cassie_batch_state_free(sb, C.c_void_p(Ss))
    d.free_state(Sd)
    b.free_state(S)
    for x in (b, c, d):
        x.close()


def test_a_smaller_batch_created_later_leaves_a_larger_ones_launches_alone(P):
    """a helper batch of another size (to prepare bank poses) shares the step instances' shared-memory limit with the batch it serves: creating a
    smaller one after a larger one must not lower the limit below the larger one's launch size"""
    big = _batch(P, 'cassie', False, 2048, seed=22)
    small = _batch(P, 'cassie', False, 16, seed=22)
    big.step(5)
    small.step(5)
    big.sync()
    small.sync()
    assert big.launch_count() >= 2 and np.isfinite(big.qpos()).all()
    for x in (big, small):
        x.close()
