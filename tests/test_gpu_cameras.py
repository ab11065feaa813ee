"""Camera sets on the H100 (cassie_batch_set_cameras, per-environment mounts, geom ids): the device rows against the fp64 camera oracle
(tests/camera_oracle.c), the one-camera path against the images the one-camera kernel rendered before camera sets existed, k cameras in one launch
against k launches, rows written through the device view against the same rows set by the verb, stepping and the model-input rules, refusals, shapes
and views.

The rig (tests/camera_set_support.py): the egocentric mount of cassie_depth.xml on the pelvis, a camera on the left tarsus looking down, a world-body
camera; per-environment rows move each camera by up to 2 cm, turn it by up to 3 degrees and change its fovy by up to 5 degrees.  fp64: z-depth within
1e-11 of the oracle (as tests/test_gpu_camera.py: the device's fused multiply-adds move body poses in their last bits).  fp32: within 1e-5 zfar
outside the pixels whose hit / miss or geom changes in the oracle when the camera moves by 1e-5 m (fewer than 0.5 %).  Geom ids: equal to the
oracle's outside those pixels."""
import ctypes as C
import os

import numpy as np
import pytest

import camera_set_support as CSS
import test_camera as TC
import test_gpu_camera as TGC
from conftest import product
from raycast_support import GOLDEN

pytestmark = pytest.mark.gpu

W, H, ZFAR = 32, 24, 4.0


def rig(P, b, model):
    q0 = TC.states(model, np.random.default_rng(0))[0]
    return CSS.rig(model, lambda name: b.name2id('body', name), q0)


def placed_stairs(b, scene0, rng, n):
    """per-environment stairs ahead of each robot of cassie.xml (as tests/test_gpu_camera.py places them)"""
    boxes = [scene0.t['names_geom'][g] for k, g in enumerate(scene0.slots) if scene0.type[k] == 6][:6]
    q = b.qpos()
    placed = {}
    for bx in boxes:
        pos = np.column_stack([q[:, 0] + rng.uniform(0.3, 2.0, n), q[:, 1] + rng.uniform(-1, 1, n), rng.uniform(-0.1, 0.15, n)])
        yaw = rng.uniform(-np.pi, np.pi, n)
        bq = np.stack([np.cos(yaw / 2), np.zeros(n), np.zeros(n), np.sin(yaw / 2)], 1)
        size = rng.uniform([0.1, 0.1, 0.05], [0.5, 0.5, 0.3], size=(n, 3))
        b.set_env_geom_pose(bx, pos=pos, quat=bq, size=size)
        placed[bx] = (pos, bq, size)
    return placed


def check_against_oracle(sim, model, b, cams, rows, envs, fp32, terrains=None, placed=None):
    depth, geom, qpos = b.depth(), b.camera_geoms(), b.qpos()
    scene0 = sim.scene()
    n_amb, n_pix, seen = 0, 0, set()
    for e in envs:
        sc = scene0
        if placed is not None:
            sc = scene0.copy()
            for gname, (p_, q_, s_) in placed.items():
                sc.place(gname, pos=p_[e], quat=q_[e], size=s_[e])
        hf = None if terrains is None else terrains[e % len(terrains)]
        for c, cam in enumerate(cams):
            r = rows[e, c]
            d, g, amb = CSS.oracle_view(sim.table, sim.moving_geoms, model, qpos[e], sc, cam[0], r[0:3], r[3:7], r[7], W, H, ZFAR, hf, amb=True)
            gm = sim.model_geom(g)
            n_amb += amb.sum()
            n_pix += W * H
            seen |= set(gm[~amb].ravel())
            assert np.array_equal(geom[e, c][~amb], gm[~amb]), (e, c, np.argwhere((geom[e, c] != gm) & ~amb)[:5])
            err = np.abs(depth[e, c] - d)[~amb].max() if fp32 else np.abs(depth[e, c] - d).max()
            assert err <= (1e-5 * ZFAR if fp32 else 1e-11), (e, c, err)
    assert n_amb < 0.005 * n_pix, n_amb / n_pix
    return seen


@pytest.mark.parametrize('model', list(TC.SETUPS))
def test_three_cameras_fp64_match_oracle(model):
    P = product()
    rng = np.random.default_rng(41)
    sim = CSS.EmuCams(model)
    terrains = None
    if model == 'cassie_hfield':
        terrains = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
        terrains[:, 95:105, 95:105] = 0
    n = 4
    b = TGC.settled_batch(P, model, n, P.FP64, terrains, ticks=300)
    placed = placed_stairs(b, sim.scene(), rng, n) if model == 'cassie' else None
    cams = rig(P, b, model)
    b.set_cameras(cams, width=W, height=H, zfar=ZFAR)
    rows = CSS.random_rows(rng, cams, n)
    b.set_env_cameras(pos=rows[..., 0:3], quat=rows[..., 3:7], fovy=rows[..., 7])
    b.enable_camera_geoms()
    b.render_depth()
    assert b.depth().shape == (n, 3, H, W) and b.camera_geoms().shape == (n, 3, H, W)
    seen = check_against_oracle(sim, model, b, cams, rows, range(n), False, terrains, placed)
    assert -1 in seen and set(sim.moving_geoms) & seen
    sim.close()
    b.close()


def test_two_cameras_fp32_4096_match_oracle():
    P = product()
    rng = np.random.default_rng(43)
    model, n = 'cassie_depth', 4096
    sim = CSS.EmuCams(model)
    b = TGC.settled_batch(P, model, n, P.FP32)
    cams = rig(P, b, model)[::2]   # the pelvis and world cameras (a camera deep in the leg chain adds the fp32 body-pose error: DESIGN.md section 3)
    b.set_cameras(cams, width=W, height=H, zfar=ZFAR)
    rows = CSS.random_rows(rng, cams, n)
    b.set_env_cameras(pos=rows[..., 0:3], quat=rows[..., 3:7], fovy=rows[..., 7])
    b.enable_camera_geoms()
    b.render_depth()
    rows32 = rows.astype(np.float32).astype(np.float64)   # what the fp32 rows hold
    check_against_oracle(sim, model, b, cams, rows32, rng.choice(n, 64, replace=False), True)
    sim.close()
    b.close()


@pytest.mark.parametrize('prec', ['fp32', 'fp64'])
def test_one_camera_is_bitwise_the_one_camera_kernel(prec):
    """set_camera and a one-camera set_cameras without rows or geom ids render the images the one-camera kernel rendered before camera sets existed
    (tests/golden/camera_set_k1_gpu.npz, recorded with that build on an H100 from the same qpos).  With geom ids the set kernel renders the same
    camera within a few ulps of depth (the device's fused multiply-adds fall differently in the two kernels) and the same geom ids the oracle gives"""
    P = product()
    G = np.load(os.path.join(GOLDEN, 'camera_set_k1_gpu.npz'))
    pr = P.FP32 if prec == 'fp32' else P.FP64
    for model, (cam, zfar) in K1_SETUPS.items():
        q = G[model + '/qpos']
        want = G['%s/%s' % (model, prec)].astype(np.float64)
        n = len(q)
        b = P.CassieBatch(n, modelfile=P.model_path(model), precision=pr)
        b.set_qpos(q)
        if isinstance(cam, str):
            b.set_camera(cam, width=W, height=H, zfar=zfar)
        else:
            body, pos, quat, fovy = cam
            b.set_camera(body=body, pos=pos, quat=quat, fovy=fovy, width=W, height=H, zfar=zfar)
        b.render_depth()
        assert np.array_equal(b.depth(), want), (model, np.abs(b.depth() - want).max())
        b.set_cameras([cam], width=W, height=H, zfar=zfar)
        b.render_depth()
        assert b.depth().shape == (n, 1, H, W) and np.array_equal(b.depth()[:, 0], want), model
        b.enable_camera_geoms()
        b.render_depth()
        ulp = np.spacing(want.astype(np.float32 if prec == 'fp32' else np.float64)).astype(np.float64)
        err = np.abs(b.depth()[:, 0] - want) / ulp
        print(model, prec, 'set kernel against the one-camera kernel: %d of %d pixels differ, at most %g ulp' % ((err > 0).sum(), err.size, err.max()))
        assert err.max() <= 4, (model, err.max())
        b.close()


K1_SETUPS = {
    'cassie_depth': ('egocentric', 4.0),
    'cassie_hfield': ('egocentric', 4.0),
    'cassie_tray_box': (('cassie-pelvis', [0.8, 0.0, 0.9], [0.921060994002885, 0.0, 0.3894183423086505, 0.0], 60.0), 3.0),
}


@pytest.mark.parametrize('prec', ['fp32', 'fp64'])
def test_one_launch_equals_separate_launches_and_device_rows_equal_verb_rows(prec):
    import torch
    P = product()
    pr = P.FP32 if prec == 'fp32' else P.FP64
    rng = np.random.default_rng(45)
    terrains = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
    n = 512
    b = TGC.settled_batch(P, 'cassie_hfield', n, pr, terrains, ticks=100)
    cams = rig(P, b, 'cassie_hfield') + ['gopro']
    b.set_cameras(cams, width=W, height=H, zfar=ZFAR)
    assert b.ncameras() == 4
    b.enable_camera_geoms()
    b.render_depth()
    d_all, g_all = b.depth(), b.camera_geoms()
    for c, cam in enumerate(cams):   # each camera alone
        b.set_cameras([cam], width=W, height=H, zfar=ZFAR)
        b.render_depth()
        assert np.array_equal(b.depth()[:, 0], d_all[:, c]) and np.array_equal(b.camera_geoms()[:, 0], g_all[:, c]), c
    # rows: set by the verb, and the same values written through the device view, render the same images
    b.set_cameras(cams, width=W, height=H, zfar=ZFAR)
    rows = CSS.random_rows(rng, cams[:3] + [b.model_camera('gopro')], n)
    b.set_env_cameras(pos=rows[..., 0:3], quat=rows[..., 3:7], fovy=rows[..., 7])
    b.render_depth()
    d_verb, g_verb = b.depth(), b.camera_geoms()
    b.clear_env_cameras()
    b.render_depth()
    assert np.array_equal(b.depth(), d_all)   # back to the set's mounts
    b.set_env_cameras()   # rows holding the set's mounts
    b.sync()
    tv = b.torch_view('camera_env')
    assert tv.shape == (n, 4, 8)
    tv.copy_(torch.as_tensor(rows, dtype=tv.dtype, device=tv.device))
    torch.cuda.synchronize()
    b.render_depth()
    assert np.array_equal(b.depth(), d_verb) and np.array_equal(b.camera_geoms(), g_verb)
    p, q, f = b.env_cameras()   # written on the device: reported from the rows
    assert np.allclose(p, rows[..., 0:3], atol=1e-6) and np.allclose(f, rows[..., 7], atol=1e-4)
    b.close()


def test_stepping_resets_snapshots_and_copy():
    P = product()
    rng = np.random.default_rng(47)
    a, c = (TGC.settled_batch(P, 'cassie_depth', 256, P.FP32, ticks=0) for _ in range(2))
    for b in (a, c):
        b.enable_aux()
    cams = rig(P, a, 'cassie_depth')
    a.set_cameras(cams, width=W, height=H, zfar=ZFAR)
    rows = CSS.random_rows(rng, cams, 256)
    a.set_env_cameras(pos=rows[..., 0:3], quat=rows[..., 3:7], fovy=rows[..., 7])
    a.enable_camera_geoms()
    for _ in range(20):
        a.render_depth()
        a.step(10)
        c.step(10)
    for f in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
        assert np.array_equal(getattr(a, f)(), getattr(c, f)()), f
    before = a.env_cameras()
    a.render_depth()
    d0 = a.depth()
    snap = a.get_state()
    a.step(20)
    a.reset()
    a.set_reset_bank(snap)
    import torch
    a.reset_where(torch.ones(256, dtype=torch.bool, device='cuda'))
    a.sync()
    a.set_state(snap)
    a.free_state(snap)
    after = a.env_cameras()
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    a.render_depth()
    assert np.array_equal(a.depth(), d0)   # the state and the rows are as before
    a.close()
    c.close()
    # cassie_sim_copy copies the rows between sets of as many cameras
    L = P.lib()
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    s1, s2 = P.CassieSim(P.model_path('cassie_depth')), P.CassieSim(P.model_path('cassie_depth'))
    b1, b2 = L.cassie_sim_batch(s1.c), L.cassie_sim_batch(s2.c)
    ip, dp = C.POINTER(C.c_int), C.POINTER(C.c_double)
    L.cassie_batch_set_cameras.argtypes = [C.c_void_p, C.c_int, ip, dp, dp, dp, C.c_int, C.c_int, C.c_double]
    L.cassie_batch_set_env_cameras.argtypes = [C.c_void_p, dp, dp, dp, C.c_void_p]
    L.cassie_batch_get_env_cameras.argtypes = [C.c_void_p, dp, dp, dp]
    body = np.array([cam[0] for cam in cams[:2]], dtype=np.int32)
    pos, quat, fovy = (np.ascontiguousarray([np.asarray(cam[i], float) for cam in cams[:2]]) for i in (1, 2, 3))
    for bb in (b1, b2):
        assert L.cassie_batch_set_cameras(bb, 2, body.ctypes.data_as(ip), pos.ctypes.data_as(dp), quat.ctypes.data_as(dp), fovy.ctypes.data_as(dp), 8, 8, 2.0) == 0
    f1 = np.ascontiguousarray([[30.0, 70.0]])
    assert L.cassie_batch_set_env_cameras(b1, None, None, f1.ctypes.data_as(dp), None) == 0
    s2.copy(s1)
    got = np.zeros((1, 2))
    assert L.cassie_batch_get_env_cameras(b2, None, None, got.ctypes.data_as(dp)) == 0
    assert np.array_equal(got, f1)


def test_refusals_shapes_and_views():
    import torch
    P = product()
    n = 16
    b = P.CassieBatch(n, modelfile=P.model_path('cassie_depth'), precision=P.FP32)
    cams = rig(P, b, 'cassie_depth')
    body, pos, quat, fovy = b.model_camera('egocentric')
    assert body == b.name2id('body', 'cassie-pelvis') and fovy == 65.5 and pos.shape == (3,) and quat.shape == (4,)
    for bad in ('nope', 'track'):
        with pytest.raises(RuntimeError):
            b.model_camera(bad)
    with pytest.raises(RuntimeError, match='no cameras are set'):
        b.set_env_cameras()
    b.set_cameras(cams, width=W, height=H, zfar=ZFAR)
    assert b.ncameras() == 3
    assert b.L.cassie_batch_row_width(b.h, b'depth') == 3 * W * H and b.L.cassie_batch_row_width(b.h, b'camera_env') == 24
    assert b.L.cassie_batch_row_width(b.h, b'camera_geom') == 3 * W * H
    b.render_depth()
    d = b.depth()
    assert d.shape == (n, 3, H, W)
    with pytest.raises(RuntimeError):
        b.camera_geoms()                 # not enabled
    with pytest.raises(RuntimeError):
        b.torch_view('camera_env')       # no rows yet
    b.enable_camera_geoms()
    with pytest.raises(RuntimeError):
        b.camera_geoms()                 # no render since
    b.render_depth()
    g = b.camera_geoms()
    b.set_env_cameras(fovy=np.full((n, 3), 50.0), mask=np.arange(n) % 2)
    p0, q0, f0 = b.env_cameras()
    b.sync()
    for field, shape in (('depth', (n, 3, H, W)), ('camera_geom', (n, 3, H, W)), ('camera_env', (n, 3, 8))):
        tv = b.torch_view(field)
        assert isinstance(tv, torch.Tensor) and tv.shape == shape, field
    assert b.torch_view('camera_geom').dtype == torch.int32
    assert np.array_equal(b.torch_view('camera_geom').cpu().numpy(), g)
    ptrs = {f: b.device_ptr(f) for f in ('depth', 'camera_geom', 'camera_env')}
    # refused sets and rows change nothing
    ok = [(c[0], c[1], c[2], c[3]) for c in cams]
    bad_sets = [ok + [ok[0], ok[0]], [(99,) + ok[0][1:]], [ok[0], (ok[1][0], ok[1][1], [0, 0, 0, 0], 60.0)], [ok[0], ok[1][:3] + (180.0,)],
                [ok[0], (ok[1][0], [np.nan, 0, 0], ok[1][2], 60.0)]]
    for cs in bad_sets:
        with pytest.raises(RuntimeError):
            b.set_cameras(cs, width=W, height=H, zfar=ZFAR)
    with pytest.raises(RuntimeError, match='camera 1'):
        b.set_cameras([ok[0], ok[1][:3] + (0.0,)], width=W, height=H, zfar=ZFAR)
    for kw in (dict(width=257), dict(height=0), dict(zfar=0.0), dict(zfar=float('inf'))):
        with pytest.raises(RuntimeError):
            b.set_cameras(ok, **{**dict(width=W, height=H, zfar=ZFAR), **kw})
    bad_rows = [dict(pos=np.full((n, 3, 3), np.nan)), dict(quat=np.zeros((n, 3, 4))), dict(fovy=np.full((n, 3), 180.0)), dict(fovy=np.zeros((n, 3)))]
    for kw in bad_rows:
        with pytest.raises(RuntimeError, match='environment 0, camera 0'):
            b.set_env_cameras(**kw)
    fv = np.full((n, 3), 50.0)
    fv[5, 2] = np.inf
    with pytest.raises(RuntimeError, match='environment 5, camera 2: fovy'):
        b.set_env_cameras(fovy=fv)
    assert b.ncameras() == 3 and all(b.device_ptr(f) == p for f, p in ptrs.items())
    p1, q1, f1 = b.env_cameras()
    assert np.array_equal(p0, p1) and np.array_equal(q0, q1) and np.array_equal(f0, f1)
    assert np.array_equal(f1[1], [50.0] * 3) and np.array_equal(f1[0], [c[3] for c in cams])
    assert np.array_equal(b.depth(), d)
    # a new set drops the rows; an empty set drops the cameras
    b.set_cameras(cams[:1], width=8, height=8, zfar=2.0)
    assert not b.device_ptr('camera_env') and not b.device_ptr('depth') and not b.device_ptr('camera_geom')
    b.render_depth()
    assert b.depth().shape == (n, 1, 8, 8) and b.camera_geoms().shape == (n, 1, 8, 8)
    b.enable_camera_geoms(False)
    assert not b.device_ptr('camera_geom')
    b.set_cameras([], width=8, height=8)
    assert b.ncameras() == 0 and b.L.cassie_batch_row_width(b.h, b'depth') == 0
    with pytest.raises(RuntimeError):
        b.render_depth()
    # set_camera keeps its shape
    b.set_camera('egocentric', width=W, height=H, zfar=ZFAR)
    b.render_depth()
    assert b.depth().shape == (n, H, W) and b.ncameras() == 1
    b.close()
