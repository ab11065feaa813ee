"""GPU: per-environment terrain (cassie_batch_set_env_hfield) -- batches in which every environment picks its own bank entry, height-field position
and size, against one oracle per sampled environment; the ray and camera kernels on the same environments; a curriculum step mid-run; the verbs'
semantics and the legacy size verbs.  CPU twins (host emulation): tests/test_env_terrain.py."""
import ctypes as C

import numpy as np
import pytest

import camera_support as CS
import raycast_support as RS
from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product
from test_env_terrain import CMODEL, SHARED_POS, SHARED_SIZE, hf_scene, oracle_on, terrain_bank

pytestmark = pytest.mark.gpu

PELVIS = 2   # cassie_hfield.xml: world, floor, cassie-pelvis


def _layout(n, K, seed):
    """random selections, elevation scales in [0, 2]x, half-extents and position offsets"""
    rng = np.random.default_rng(seed)
    t = rng.integers(0, K, n).astype(np.int32)
    pos = SHARED_POS + rng.uniform(-0.05, 0.05, (n, 3))
    size = np.stack([rng.uniform(3.5, 6.0, n), rng.uniform(3.5, 6.0, n), SHARED_SIZE[2] * rng.uniform(0, 2, n), np.full(n, SHARED_SIZE[3])], axis=1)
    return t, pos, size


def _pushes(n, seed):
    return np.concatenate([np.random.default_rng(seed).uniform(-40, 40, (n, 2)), np.zeros((n, 4))], axis=1)


@pytest.mark.parametrize('fp64', [False, True])
def test_per_env_terrain_follows_the_oracle(oracle_mod, fp64):
    """a 64-terrain bank, random selections, scales, sizes and positions, PD standing with pushes, 600 ticks; 64 sampled environments replayed by the
    oracle, then their height scans and depth images against the ray and camera oracles at the batch's state"""
    P, O = product(), oracle_mod
    n, K = (256, 64) if fp64 else (4096, 64)
    bank = terrain_bank(K, 41)
    t, pos, size = _layout(n, K, 5)
    b = P.CassieBatch(n, modelfile=CMODEL, precision=P.FP64 if fp64 else P.FP32)
    b.set_hfield_data(bank)
    b.set_env_hfield(terrain=t, pos=pos, size=size)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    sample = np.random.default_rng(8).choice(n, 64, replace=False)
    oracles = [oracle_on(O, bank[t[e]], pos[e], size[e]) for e in sample]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    push = _pushes(n, 9)
    iters_ok = True
    for k in range(600):
        if k in (200, 260):
            on = k == 200
            b.apply_force(push if on else np.zeros((n, 6)))
            for e, o in zip(sample, oracles):
                o.arr('xfrc_applied').reshape(-1, 6)[PELVIS] = push[e] if on else 0
        b.step(1)
        for o in oracles:
            o.step_pd(u)
        if fp64 and k % 50 == 49:
            it = b.counters()[sample, 3]
            iters_ok = iters_ok and all(int(it[i]) == o.get_int('solver_iter') for i, o in enumerate(oracles))
    q = b.qpos()
    err = np.array([np.abs(q[e] - o.arr('qpos')).max() for e, o in zip(sample, oracles)])
    print('qpos error vs oracle: median %.3g p90 %.3g worst %.3g' % (np.median(err), np.percentile(err, 90), err.max()))
    if fp64:
        assert err.max() <= 1e-9 and iters_ok, err.max()
    else:
        assert np.median(err) <= 1e-5 and np.percentile(err, 90) <= 1e-4 and err.max() <= 1e-3
    assert int(b.counters()[:, 4].sum()) == 0
    # height scans: the heading-frame grid around the pelvis; depth images: the model's egocentric camera
    xs, ys = np.linspace(-1.0, 1.0, 11), np.linspace(-0.6, 0.6, 7)
    b.set_height_scan(xs, ys, z_start=1.0, max_dist=3.0)
    b.raycast()
    rays = b.rays()
    body, cpos, cquat, fovy, mode = CS.cameras_fixture()[('cassie_hfield', 'egocentric')]
    W, H, zfar = 24, 18, 4.0
    b.set_camera(name='egocentric', width=W, height=H, zfar=zfar)
    b.render_depth()
    depth = b.depth()
    cam = CS.EmuCam('cassie_hfield')
    sc0, bid = cam.scene(), cam.body(body)
    org, dirs = RS.height_scan(xs, ys, 1.0)
    for e in sample[:16]:
        xpos, xquat = CS.oracle_poses('cassie_hfield', q[e])
        ow, dw = RS.world_rays(RS.HEADING, org, dirs, xpos[3 * PELVIS:3 * PELVIS + 3], RS.quat2mat(xquat[4 * PELVIS:4 * PELVIS + 4]))
        sc, hf = hf_scene(sc0, pos[e], size[e]), bank[t[e]].astype(np.float64)
        ref = RS.oracle_cast(sc, ow, dw, 3.0, hf)
        mv = CS.Moving(cam.table, cam.moving_geoms, xpos, xquat)
        cp, cR = CS.camera_world(xpos, xquat, bid, np.asarray(cpos, float), np.asarray(cquat, float) / np.linalg.norm(cquat))
        img, _ = CS.oracle_render(sc, mv, cp, cR, fovy, W, H, zfar, hf)
        if fp64:   # depth: 1e-11, as tests/test_gpu_camera.py (the device's fused multiply-adds move the composed body poses in their last bits)
            assert np.abs(rays[e][:, :2] - ref[:, :2]).max() <= 1e-12 and np.array_equal(rays[e][:, 2], ref[:, 2]) and np.abs(depth[e] - img).max() <= 1e-11, e
        else:
            amb = RS.ambiguous(sc, ow, dw, 3.0, hf)
            assert np.array_equal(rays[e][~amb, 2], ref[~amb, 2]) and np.abs(rays[e][~amb] - ref[~amb]).max() <= 1e-5 * 3.0, e
            pa = CS.ambiguous(sc, mv, cp, cR, fovy, W, H, zfar, hf)
            assert np.abs(depth[e] - img)[~pa].max() <= 1e-5 * zfar, e
    cam.close()


@pytest.mark.parametrize('fp64', [False, True])
def test_default_rows_are_bitwise_no_rows(fp64):
    """selections e % K with the shared position and size: qpos, qvel, obs, aux and the counters bitwise those of the batch without rows"""
    P = product()
    n, K = 512, 8
    bank = terrain_bank(K, 2)
    a, b = (P.CassieBatch(n, modelfile=CMODEL, precision=P.FP64 if fp64 else P.FP32) for _ in range(2))
    for x in (a, b):
        x.set_hfield_data(bank)
        x.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
        x.enable_aux(True)
    b.set_env_hfield(terrain=np.arange(n) % K, pos=SHARED_POS, size=SHARED_SIZE)
    push = _pushes(n, 3)
    for k in range(6):
        for x in (a, b):
            x.apply_force(push if k % 2 else np.zeros((n, 6)))
            x.step(50)
        for f in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
            assert np.array_equal(getattr(a, f)(), getattr(b, f)()), (k, f)


def test_curriculum_step_mid_run(oracle_mod):
    """mid-run, masked environments get a new terrain and scale (the selection once through the verb, once through torch_view('terrain')) and a masked
    restore of the starting state: they follow an oracle started from that state on their new terrain; the other environments are bitwise unaffected"""
    import torch
    P, O = product(), oracle_mod
    n, K = 64, 8
    bank = terrain_bank(K, 13)
    t, pos, size = _layout(n, K, 6)
    b, twin = (P.CassieBatch(n, modelfile=CMODEL, precision=P.FP64) for _ in range(2))
    for x in (b, twin):
        x.set_hfield_data(bank)
        x.set_env_hfield(terrain=t, pos=pos, size=size)
        x.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    s0 = b.get_state()
    for x in (b, twin):
        x.step(300)
    mask = np.zeros(n, dtype=np.uint8)
    mask[::4] = 1
    t2, size2 = (t + 3) % K, size * [1, 1, 0, 1] + [0, 0, 0.35, 0]
    via_verb = mask.copy()
    via_verb[::8] = 0   # every other masked environment gets its selection through the device row instead
    b.set_env_hfield(terrain=t2, mask=via_verb)
    b.set_env_hfield(size=size2, mask=mask)
    view = b.torch_view('terrain')
    assert view.dtype == torch.int32 and view.shape == (n,)
    rows = torch.as_tensor(np.flatnonzero(mask & ~via_verb), device=view.device)
    view[rows] = torch.as_tensor(t2, device=view.device)[rows]
    torch.cuda.synchronize()
    b.set_state(s0, mask)
    assert np.array_equal(b.env_hfield()[0], np.where(mask == 1, t2, t))
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    moved = np.flatnonzero(mask)
    oracles = [oracle_on(O, bank[t2[e]], pos[e], size2[e]) for e in moved]
    for k in range(300):
        b.step(1)
        twin.step(1)
        for o in oracles:
            o.step_pd(u)
    q, qt = b.qpos(), twin.qpos()
    err = max(np.abs(q[e] - o.arr('qpos')).max() for e, o in zip(moved, oracles))
    assert err <= 1e-9, err
    keep = mask == 0
    assert np.array_equal(q[keep], qt[keep]) and np.array_equal(b.qvel()[keep], twin.qvel()[keep]) and np.array_equal(b.obs()[keep], twin.obs()[keep])
    b.free_state(s0)


def test_verb_semantics():
    P = product()
    n, K = 16, 4
    bank = terrain_bank(K, 21)
    b = P.CassieBatch(n, modelfile=CMODEL, precision=P.FP32)
    b.set_hfield_data(bank)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    t0, pos0, size0 = b.env_hfield()
    assert np.array_equal(t0, np.arange(n) % K) and np.allclose(pos0, SHARED_POS) and np.allclose(size0, SHARED_SIZE)
    t, pos, size = _layout(n, K, 1)
    b.set_env_hfield(terrain=t, pos=pos, size=size)
    before = b.env_hfield()
    bad_t = t.copy()
    bad_t[3] = K
    for kw, word in ((dict(terrain=bad_t), 'terrain'), (dict(terrain=np.full(n, -1)), 'terrain'), (dict(size=[0, 1, 0.1, 0.1]), 'size'),
                     (dict(size=[1, 1, -0.1, 0.1]), 'size'), (dict(size=[1, 1, 0.1, -1]), 'size'), (dict(pos=[0, np.nan, 0]), 'pos'),
                     (dict(size=[1, np.inf, 0.1, 0.1]), 'size')):
        with pytest.raises(RuntimeError) as ex:
            b.set_env_hfield(**kw)
        assert 'environment' in str(ex.value) and word in str(ex.value), str(ex.value)
        for x, y in zip(before, b.env_hfield()):
            assert np.array_equal(x, y)
    with pytest.raises(RuntimeError):
        b.set_hfield_size([1, 0, 0.1, 0.1])
    plain = P.CassieBatch(2, precision=P.FP32)
    with pytest.raises(RuntimeError, match='height field'):
        plain.set_env_hfield(terrain=[0, 0])
    # a value >= K written to the device row reads entry t % K
    c = P.CassieBatch(n, modelfile=CMODEL, precision=P.FP32)
    c.set_hfield_data(bank)
    c.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    c.set_env_hfield(terrain=t, pos=pos, size=size)
    import torch
    v = c.torch_view('terrain')
    v += torch.as_tensor(K * (np.arange(n) % 3 + 1), device=v.device, dtype=torch.int32)
    torch.cuda.synchronize()
    # reset and snapshot restore leave the rows alone
    s = b.get_state()
    b.step(100)
    c.step(100)
    assert np.array_equal(b.qpos(), c.qpos())
    b.reset()
    b.set_state(s)
    b.free_state(s)
    for x, y in zip(before, b.env_hfield()):
        assert np.array_equal(x, y)
    # a new bank with another K keeps the selections; they are read mod the new K
    b.set_hfield_data(bank[:3])
    assert np.array_equal(b.env_hfield()[0], t)
    d = P.CassieBatch(n, modelfile=CMODEL, precision=P.FP32)
    d.set_hfield_data(bank[:3])
    d.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    d.set_env_hfield(terrain=t % 3, pos=pos, size=size)
    b.reset()
    d.reset()
    b.step(100)
    d.step(100)
    assert np.array_equal(b.qpos(), d.qpos())
    # the shared size: position and size back to the shared ones, selections stay; clear: back to e % K
    b.set_hfield_size([4.0, 4.0, 0.3, 0.1])
    tt, pp, ss = b.env_hfield()
    assert np.array_equal(tt, t) and np.allclose(pp, SHARED_POS) and np.allclose(ss, [4.0, 4.0, 0.3, 0.1]) and np.allclose(b.hfield_size(), [4.0, 4.0, 0.3, 0.1])
    b.set_env_hfield(pos=pos, size=size)
    b.clear_env_geom_poses()   # also returns the height field's position and size to the shared ones, keeps the selections
    tt, pp, ss = b.env_hfield()
    assert np.array_equal(tt, t) and np.allclose(pp, SHARED_POS) and np.allclose(ss, [4.0, 4.0, 0.3, 0.1])
    b.clear_env_hfield()
    assert np.array_equal(b.env_hfield()[0], np.arange(n) % 3)


def test_legacy_size_verbs(oracle_mod):
    """CassieSim.set_hfield_size with twice the elevation scale follows the oracle with that size; a write through the borrowed pointer takes effect at
    the next step; cassie_sim_copy carries the size; a model without a height field gets an error"""
    P, O = product(), oracle_mod
    data = terrain_bank(1, 31)[0]
    size = SHARED_SIZE * [1, 1, 2, 1]
    sim = P.CassieSim(modelfile=CMODEL)
    sim.L.cassie_sim_hfielddata.argtypes = [C.c_void_p]
    sim.L.cassie_sim_hfielddata.restype = C.POINTER(C.c_float)
    assert np.allclose(sim.get_hfield_size(), SHARED_SIZE)
    ptr = sim.L.cassie_sim_hfielddata(sim.c)
    C.memmove(ptr, np.ascontiguousarray(data).ctypes.data, data.nbytes)
    sim.set_hfield_size(size)
    assert np.allclose(sim.get_hfield_size(), size)
    o = oracle_on(O, data, SHARED_POS, size)
    u = P.pd_in_t()
    for leg, off in ((u.leftLeg, 0), (u.rightLeg, 5)):
        for i in range(5):
            leg.motorPd.pTarget[i] = PD_TARGET[off + i]; leg.motorPd.pGain[i] = PD_PGAIN[i]; leg.motorPd.dGain[i] = PD_DGAIN[i]
    uo = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for _ in range(500):
        sim.step_pd(u)
        o.step_pd(uo)
    assert np.abs(sim.qpos()[:35] - o.arr('qpos')).max() <= 1e-8
    # through the borrowed pointer
    a, b = P.CassieSim(modelfile=CMODEL), P.CassieSim(modelfile=CMODEL)
    sim.L.cassie_sim_get_hfield_size(a.c)[2] = 0.4
    b.set_hfield_size([5, 5, 0.4, 0.1])
    for x in (a, b):
        C.memmove(x.L.cassie_sim_hfielddata(x.c), np.ascontiguousarray(data).ctypes.data, data.nbytes)
        for _ in range(300):
            x.step_pd(u)
    assert np.array_equal(a.qpos(), b.qpos())
    ref = P.CassieSim(modelfile=CMODEL)
    C.memmove(ref.L.cassie_sim_hfielddata(ref.c), np.ascontiguousarray(data).ctypes.data, data.nbytes)
    for _ in range(300):
        ref.step_pd(u)
    assert np.abs(ref.qpos() - a.qpos()).max() > 1e-4   # the new scale was really used
    # an invalid size is not uploaded: the last valid one stays
    b.set_hfield_size([5, 5, -1, 0.1])
    b.step_pd(u)
    assert 'size' in P._last_error()
    # cassie_sim_copy carries the size
    dup = P.CassieSim(modelfile=CMODEL)
    sim.L.cassie_sim_copy.argtypes = [C.c_void_p, C.c_void_p]
    sim.L.cassie_sim_copy(dup.c, a.c)
    assert np.allclose(dup.get_hfield_size(), [5, 5, 0.4, 0.1])
    plain = P.CassieSim()
    with pytest.raises(RuntimeError, match='height field'):
        plain.get_hfield_size()
