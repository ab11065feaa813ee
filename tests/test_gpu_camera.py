"""Depth camera on the H100 (cassie_batch_render_depth): the device rows against the fp64 camera oracle (tests/camera_oracle.c) at each sampled
environment's own state, placement and terrain; rendering leaves stepping bitwise unchanged; the verbs' semantics and error cases.

Setups: the egocentric camera of cassie_depth.xml; the same camera of cassie_hfield.xml over the 64-terrain bank; a camera mounted on cassie.xml's
pelvis over per-environment stairs; a camera aimed at the tray and cup of cassie_tray_box.xml.  Batches of 4096 fp32 and 256 fp64 environments after
600 ticks under the PD controller with pushes.  fp64: z-depth within 1e-11 (the device's fused multiply-adds move body poses in their
last bits, and a hit near a silhouette magnifies that; the host emulation holds 1e-12).  fp32: within 1e-5 zfar on every pixel whose hit / miss or geom does not
change in the oracle when the camera moves by 1e-5 m in x or y (fewer than 0.5 % of the sampled pixels)."""
import ctypes as C

import numpy as np
import pytest

import camera_support as CS
import test_camera as TC
from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, product

pytestmark = pytest.mark.gpu

W, H = 32, 24


def settled_batch(P, name, n, prec, terrains=None, ticks=600):
    b = P.CassieBatch(n, modelfile=P.model_path(name), precision=prec)
    if terrains is not None:
        b.set_hfield_data(terrains)
    b.set_pd(P.pd_rows(n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))
    rng = np.random.default_rng(1)
    q = b.qpos()
    q[:, 0:2] += rng.uniform(-2, 2, size=(n, 2))
    yaw = rng.uniform(-np.pi, np.pi, n)
    q[:, 3], q[:, 4], q[:, 5], q[:, 6] = np.cos(yaw / 2), 0, 0, np.sin(yaw / 2)
    b.set_qpos(q)
    b.forward()
    for k in range(3):   # pushes: a kick of the pelvis velocity every 200 ticks
        v = b.qvel()
        v[:, 0:3] += rng.normal(size=(n, 3)) * [0.6, 0.6, 0.2]
        b.set_qvel(v)
        b.step(ticks // 3)
    return b


def camera_args(model, b):
    cam, zfar = TC.SETUPS[model]
    if isinstance(cam, str):
        b.set_camera(cam, width=W, height=H, zfar=zfar)
        body, pos, quat, fovy, _ = CS.cameras_fixture()[(model, cam)]
    else:
        body, pos, quat, fovy = cam
        b.set_camera(body=body, pos=pos, quat=quat, fovy=fovy, width=W, height=H, zfar=zfar)
    return body, np.asarray(pos, float), np.asarray(quat, float) / np.linalg.norm(quat), fovy, zfar


CASES = [(m, 4096, 'fp32') for m in TC.SETUPS] + [(m, 256, 'fp64') for m in TC.SETUPS]


@pytest.mark.parametrize('model,n,prec', CASES)
def test_depth_matches_oracle(model, n, prec):
    P = product()
    fp32 = prec == 'fp32'
    rng = np.random.default_rng(11)
    sim = CS.EmuCam(model)   # slot maps and the model table
    scene0 = sim.scene()
    terrains = None
    if model == 'cassie_hfield':   # bench.py config 4's kind: 64 terrains, a flat centre patch
        terrains = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
        terrains[:, 95:105, 95:105] = 0
    b = settled_batch(P, model, n, P.FP32 if fp32 else P.FP64, terrains)
    placed = None
    if model == 'cassie':   # per-environment stairs ahead of each robot
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
    body, pos, quat, fovy, zfar = camera_args(model, b)
    bid = sim.body(body)
    b.render_depth()
    depth, qpos = b.depth(), b.qpos()
    assert depth.shape == (n, H, W)
    n_amb, n_pix, n_mov = 0, 0, 0
    for e in rng.choice(n, 64, replace=False):
        sc = scene0
        if placed is not None:
            sc = scene0.copy()
            for gname, (p_, q_, s_) in placed.items():
                sc.place(gname, pos=p_[e], quat=q_[e], size=s_[e])
        xpos, xquat = CS.oracle_poses(model, qpos[e])
        mv = CS.Moving(sim.table, sim.moving_geoms, xpos, xquat)
        cpos, cR = CS.camera_world(xpos, xquat, bid, pos, quat)
        hf = None if terrains is None else terrains[e % 64]
        ref, g = CS.oracle_render(sc, mv, cpos, cR, fovy, W, H, zfar, hf)
        n_mov += (g >= 100).sum()
        n_pix += W * H
        if not fp32:
            assert np.abs(depth[e] - ref).max() <= 1e-11, (e, np.abs(depth[e] - ref).max())
            continue
        amb = CS.ambiguous(sc, mv, cpos, cR, fovy, W, H, zfar, hf)
        n_amb += amb.sum()
        assert np.abs(depth[e] - ref)[~amb].max() <= 1e-5 * zfar, (e, np.abs(depth[e] - ref)[~amb].max())
    assert n_amb < 0.005 * n_pix
    if model in ('cassie', 'cassie_tray_box'):
        assert n_mov > 0
    sim.close()
    b.close()


@pytest.mark.parametrize('prec', ['fp32', 'fp64'])
def test_rendering_does_not_change_stepping(prec):
    P = product()
    pr = P.FP32 if prec == 'fp32' else P.FP64
    terrains = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
    a, c = (settled_batch(P, 'cassie_hfield', 512, pr, terrains, ticks=0) for _ in range(2))
    for b in (a, c):
        b.enable_aux()
        b.set_frames(['cassie-pelvis', 'left-foot'])
    a.set_camera('egocentric', width=64, height=48, zfar=5.0)
    for t in range(50):
        a.render_depth()
        a.step(10)
        c.step(10)
    for f in ('qpos', 'qvel', 'obs', 'aux', 'frames', 'counters'):
        assert np.array_equal(getattr(a, f)(), getattr(c, f)()), f
    a.close()
    c.close()


def test_verbs_and_errors():
    import torch
    P = product()
    b = P.CassieBatch(64, modelfile=P.model_path('cassie_depth'), precision=P.FP32)
    with pytest.raises(RuntimeError):
        b.render_depth()                                  # no camera
    b.set_camera('egocentric', width=40, height=30, zfar=4.0)
    assert b.L.cassie_batch_row_width(b.h, b'depth') == 1200
    with pytest.raises(RuntimeError):
        b.depth()                                         # -1 before the first render
    with pytest.raises(RuntimeError):
        b.torch_view('depth')                             # no rows yet
    b.render_depth()
    d = b.depth()
    assert d.shape == (64, 30, 40) and (d > 0).all() and (d <= 4.0).all() and (d < 4.0).mean() > 0.3
    b.L.cassie_batch_get_depth.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    assert b.L.cassie_batch_get_depth(b.h, None) == -1   # NULL output
    b.sync()
    tv = b.torch_view('depth')
    assert isinstance(tv, torch.Tensor) and tv.shape == (64, 30, 40)
    assert np.array_equal(tv.cpu().numpy().astype(np.float64), d)
    ptr = b.device_ptr('depth')
    # bad sets return -1 and leave the camera and the rows alone
    bad = [dict(name='nope'), dict(name='track'), dict(body='nope'), dict(body='cassie-pelvis', fovy=0.0), dict(body='cassie-pelvis', fovy=180.0),
           dict(body='cassie-pelvis', width=257), dict(body='cassie-pelvis', height=0), dict(body='cassie-pelvis', width=-1),
           dict(body='cassie-pelvis', zfar=0.0), dict(body='cassie-pelvis', zfar=float('inf')), dict(body='cassie-pelvis', quat=[0, 0, 0, 0]),
           dict(body='cassie-pelvis', quat=[float('nan'), 0, 0, 1])]
    for kw in bad:
        args = dict(width=8, height=8, zfar=2.0)
        args.update(kw)
        with pytest.raises(RuntimeError):
            b.set_camera(**args)
        assert b.device_ptr('depth') == ptr and b.L.cassie_batch_row_width(b.h, b'depth') == 1200
        assert np.array_equal(b.depth(), d)
    with pytest.raises(RuntimeError, match='egocentric, gopro'):
        b.set_camera('nope', width=8, height=8)           # the message lists the model's cameras
    # rows survive reset and a snapshot restore
    snap = b.get_state()
    b.step(20)
    b.reset()
    b.set_state(snap)
    b.free_state(snap)
    assert np.array_equal(b.depth(), d)
    # a mounted camera equal to the model's egocentric camera renders the same image
    _, pos, quat, fovy, _ = CS.cameras_fixture()[('cassie_depth', 'egocentric')]
    b.set_camera(body='cassie-pelvis', pos=pos, quat=quat * 3.0, fovy=fovy, width=40, height=30, zfar=4.0)
    b.render_depth()
    assert np.abs(b.depth() - d).max() <= 1e-5
    # width 0 drops the camera
    b.set_camera(width=0)
    assert b.L.cassie_batch_row_width(b.h, b'depth') == 0 and not b.device_ptr('depth')
    with pytest.raises(RuntimeError):
        b.render_depth()
    b.close()
