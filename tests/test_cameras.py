"""Camera sets on the CPU (DESIGN.md section 3, "Depth-camera rules"): several cameras per launch, per-environment mounts and geom ids, with the camera
source compiled with -DCASSIE_EMU (tests/emu/emu_cameras.cpp).

1. A set of one camera without mount rows renders bitwise what the one-camera source rendered before camera sets existed: the images of
   tests/golden/camera_set_k1.npz, rendered from the same inputs by that source (fp64 and fp32, the four models of test_camera.py).
2. Three cameras -- the egocentric mount on the pelvis, a camera on the left tarsus looking down, a world-body camera -- with random per-environment
   mounts (position +-2 cm, rotation +-3 degrees, fovy +-5 degrees) against the fp64 camera oracle (tests/camera_oracle.c), per environment and camera,
   on cassie with per-environment stairs, cassie_depth, cassie_hfield over a terrain bank and cassie_tray_box: fp64 depth within 1e-12, fp32 within
   1e-5 zfar outside the ambiguous pixels (< 0.5 %), and geom ids equal to the oracle's outside those pixels.
3. k cameras in one pass equal k one-camera passes bitwise, with and without rows and geom ids.
4. Rows holding the set's mounts render the set's images within one ulp of depth (the kernel normalises the quaternion and forms tan(fovy / 2) itself).
5. A row the kernel cannot use (non-finite, zero quaternion, fovy outside (0, 180)) renders nothing for that camera and leaves the others alone.
"""
import os

import numpy as np
import pytest

import camera_set_support as CSS
import test_camera as TC
import test_raycast as TR
from raycast_support import GOLDEN

W, H = 24, 18
MODELS = list(TC.SETUPS)
ZFAR = 4.0


def golden():
    return np.load(os.path.join(GOLDEN, 'camera_set_k1.npz'))


# ------------------------------------------------------------------ 1. one camera, no rows: the one-camera images, bit for bit
@pytest.mark.parametrize('fp32', [False, True])
@pytest.mark.parametrize('model', MODELS)
def test_one_camera_is_bitwise_the_one_camera_source(model, fp32):
    G = golden()
    sim = CSS.EmuCams(model, fp32)
    cam = G[model + '/cam']
    body, pos, quat, fovy, zfar = int(cam[0]), cam[1:4], cam[4:8], float(cam[8]), float(cam[9])
    qs = G[model + '/qpos']
    genv = G[model + '/genv'] if model + '/genv' in G else None
    want = G['%s/%s' % (model, 'fp32' if fp32 else 'fp64')].astype(np.float64)
    got = sim.render_set([(body, pos, quat, fovy)], W, H, zfar, n=len(qs), qpos=qs, genv=genv)
    assert got.shape == (len(qs), 1, H, W)
    assert np.array_equal(got[:, 0], want), np.abs(got[:, 0] - want).max()
    got_geoms = sim.render_set([(body, pos, quat, fovy)], W, H, zfar, n=len(qs), qpos=qs, genv=genv, geoms=True)[0]
    assert np.array_equal(got_geoms, got)   # geom ids change no depth
    assert np.array_equal(sim.render(body, pos, quat, fovy, W, H, zfar, n=len(qs), qpos=qs, genv=genv), want)   # the one-camera entry
    sim.close()


# ------------------------------------------------------------------ 2. three cameras with random rows against the oracle
def scene_inputs(sim, model, qs, rng):
    n = len(qs)
    sc0 = sim.scene()
    scenes, genv, bank = [sc0] * n, None, None
    if model == 'cassie':
        scenes = [TR.stairs_scene(sim, rng) for _ in range(n)]
        for sc, q in zip(scenes, qs):
            for k, g in enumerate(sc.slots):
                if sc.type[k] == 6:
                    sc.pos[k][:2] += q[:2] + [1.2, 0]
        genv = np.array([s.genv_row() for s in scenes])
    if model == 'cassie_hfield':
        bank = np.stack([TR.terrain(rng, sc0) * 0.6 for _ in range(4)])
    return scenes, genv, bank


@pytest.mark.parametrize('fp32', [False, True])
@pytest.mark.parametrize('model', MODELS)
def test_three_cameras_with_rows_match_oracle(model, fp32):
    rng = np.random.default_rng(31)
    sim = CSS.EmuCams(model, fp32)
    qs = TC.states(model, rng)
    n = len(qs)
    cams = CSS.rig(model, sim.body, qs[0])
    rows = CSS.random_rows(rng, cams, n)
    scenes, genv, bank = scene_inputs(sim, model, qs, rng)
    depth, geom = sim.render_set(cams, W, H, ZFAR, n=n, qpos=np.array(qs), genv=genv, bank=bank, cenv=rows, geoms=True)
    n_amb, n_pix, seen = 0, 0, set()
    for e in range(n):
        hf = None if bank is None else bank[e % 4]
        for c, cam in enumerate(cams):
            r = rows[e, c]
            d, g, amb = CSS.oracle_view(sim.table, sim.moving_geoms, model, qs[e], scenes[e], cam[0], r[0:3], r[3:7], r[7], W, H, ZFAR, hf, amb=True)
            gm = sim.model_geom(g)
            n_amb += amb.sum()
            n_pix += W * H
            seen |= set(gm[~amb].ravel())
            assert np.array_equal(geom[e, c][~amb], gm[~amb]), (e, c, np.argwhere((geom[e, c] != gm) & ~amb)[:5])
            if fp32:
                assert np.abs(depth[e, c] - d)[~amb].max() <= 1e-5 * ZFAR, (e, c, np.abs(depth[e, c] - d)[~amb].max())
            else:
                assert np.abs(depth[e, c] - d).max() <= 1e-12, (e, c, np.abs(depth[e, c] - d).max())
    assert n_amb < 0.005 * n_pix, n_amb / n_pix
    assert -1 in seen and any(g >= 0 for g in seen)
    assert set(sim.moving_geoms) & seen   # the robot is in some view (the tarsus and world cameras see the legs)
    sim.close()


# ------------------------------------------------------------------ 3. k in one pass = k single passes
@pytest.mark.parametrize('fp32', [False, True])
@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield'])
def test_k_cameras_in_one_pass_equal_single_passes(model, fp32):
    rng = np.random.default_rng(5)
    sim = CSS.EmuCams(model, fp32)
    qs = TC.states(model, rng)
    n = len(qs)
    cams = CSS.rig(model, sim.body, qs[0])
    cams.append((sim.body('right-tarsus'), np.array([0.05, 0.02, 0.0]), np.array([0.3, 0.2, -0.9, 0.1]), 100.0))   # a fourth: CAM_MAX
    rows = CSS.random_rows(rng, cams, n)
    _, genv, bank = scene_inputs(sim, model, qs, rng)
    for cenv in (None, rows):
        d, g = sim.render_set(cams, W, H, ZFAR, n=n, qpos=np.array(qs), genv=genv, bank=bank, cenv=cenv, geoms=True)
        for c, cam in enumerate(cams):
            d1, g1 = sim.render_set([cam], W, H, ZFAR, n=n, qpos=np.array(qs), genv=genv, bank=bank, cenv=None if cenv is None else cenv[:, c:c + 1],
                                    geoms=True)
            assert np.array_equal(d[:, c], d1[:, 0]) and np.array_equal(g[:, c], g1[:, 0]), c
    assert sim.render_set(cams + [cams[0]], W, H, ZFAR, n=n) is None   # five cameras: refused
    sim.close()


# ------------------------------------------------------------------ 4. rows holding the set's mounts
@pytest.mark.parametrize('fp32', [False, True])
@pytest.mark.parametrize('model', MODELS)
def test_rows_holding_the_mounts_give_the_shared_images(model, fp32):
    rng = np.random.default_rng(8)
    sim = CSS.EmuCams(model, fp32)
    qs = TC.states(model, rng)
    n = len(qs)
    cams = CSS.rig(model, sim.body, qs[0])
    rows = np.array([[np.concatenate([p, np.asarray(q) / np.linalg.norm(q), [f]]) for _, p, q, f in cams]] * n)
    _, genv, bank = scene_inputs(sim, model, qs, rng)
    a, ga = sim.render_set(cams, W, H, ZFAR, n=n, qpos=np.array(qs), genv=genv, bank=bank, geoms=True)
    b, gb = sim.render_set(cams, W, H, ZFAR, n=n, qpos=np.array(qs), genv=genv, bank=bank, cenv=rows, geoms=True)
    dt = np.float32 if fp32 else np.float64
    ulp = np.spacing(a.astype(dt)).astype(np.float64)
    assert (np.abs(a - b) <= ulp).all(), np.abs(a - b).max()
    same = a == b
    assert np.array_equal(ga[same], gb[same])
    assert same.mean() > 0.99
    sim.close()


# ------------------------------------------------------------------ 5. rows the kernel cannot use
@pytest.mark.parametrize('fp32', [False, True])
def test_unusable_rows_render_nothing(fp32):
    rng = np.random.default_rng(2)
    sim = CSS.EmuCams('cassie_depth', fp32)
    qs = TC.states('cassie_depth', rng)
    cams = CSS.rig('cassie_depth', sim.body, qs[0])
    rows = CSS.random_rows(rng, cams, 1)
    base, gbase = sim.render_set(cams, W, H, ZFAR, n=1, qpos=np.array(qs[:1]), cenv=rows, geoms=True)
    assert (gbase[0, 0] >= 0).mean() > 0.3
    for f, v in ((0, np.nan), (2, np.inf), (3, 0.0), (4, np.nan), (7, 0.0), (7, 180.0), (7, -5.0), (7, np.nan)):
        bad = rows.copy()
        bad[0, 0, f] = v
        if f == 3:
            bad[0, 0, 3:7] = 0
        d, g = sim.render_set(cams, W, H, ZFAR, n=1, qpos=np.array(qs[:1]), cenv=bad, geoms=True)
        assert (d[0, 0] == ZFAR).all() and (g[0, 0] == -1).all(), (f, v)
        assert np.array_equal(d[0, 1:], base[0, 1:]) and np.array_equal(g[0, 1:], gbase[0, 1:])
    sim.close()
