"""Depth camera on the CPU (DESIGN.md section 3, "Depth camera").

1. The fp64 camera oracle (tests/camera_oracle.c) against an independent numpy statement: the ray oracle's numpy twin for the static geoms, and for
   the moving geoms a sphere quadratic, a slab test and a capsule taken as the union of its cylinder and two whole end spheres; random scenes with
   hits from outside, cameras inside geoms, grazes and capsule caps: z-depths within 1e-12, equal geoms.
2. The camera source compiled with -DCASSIE_EMU (tests/emu/emu_camera.cpp) against the oracle at standing, mid-fall and crossed-leg states of the fp64
   oracle stepper, on cassie_depth (egocentric), cassie_hfield with 4 terrains, cassie with a mounted camera and per-environment stairs, and
   cassie_tray_box with a camera aimed at the tray and cup: fp64 within 1e-12, fp32 within 1e-5 zfar outside ambiguous pixels (< 0.5 %).
3. The body poses the camera source composes equal the step source's frame rows after a forward (fp64, 1e-15).
4. Known geometry over a flat floor: straight down reads the height on every pixel, a tilted camera the analytic plane depth.
5. The camera is checked before anything is rendered.
"""
import os

import numpy as np
import pytest

import camera_support as CS
import oracle as O
import raycast_support as RS
import test_raycast as TR

G = RS.GOLDEN


# ------------------------------------------------------------------ 1. oracle vs numpy
def pixel_rays(cpos, cR, fovy, W, H):
    ty = np.tan(np.radians(fovy) / 2)
    tx = ty * W / H
    c, r = np.meshgrid(np.arange(W), np.arange(H))
    dc = np.stack([(2 * (c + 0.5) / W - 1) * tx, (1 - 2 * (r + 0.5) / H) * ty, -np.ones_like(c, dtype=float)], -1).reshape(-1, 3)
    nd = np.linalg.norm(dc, axis=1)
    return np.tile(cpos, (len(dc), 1)), (dc @ cR.T) / nd[:, None], nd


def np_sphere(c, r, o, d):
    w = o - c
    b, cc = w @ d, w @ w - r * r
    disc = b * b - cc
    if cc <= 0 or disc < 0:
        return np.inf
    t = -b - np.sqrt(disc)
    return t if t > 0 else np.inf


def np_moving(ty, p, R, s, o, d):
    lo, ld = R.T @ (o - p), R.T @ d
    if ty == 2:
        return np_sphere(p, s[0], o, d)
    if ty == 6:
        if np.all(np.abs(lo) < s):
            return np.inf
        with np.errstate(divide='ignore', invalid='ignore'):
            a, b = (-s - lo) / ld, (s - lo) / ld
        par = ld == 0
        if np.any(par & (np.abs(lo) > s)):
            return np.inf
        t0 = np.max(np.where(par, -np.inf, np.minimum(a, b)))
        t1 = np.min(np.where(par, np.inf, np.maximum(a, b)))
        return t0 if (t1 >= t0 and t0 > 0) else np.inf
    r, h = s[0], s[1]
    ends = [p + R[:, 2] * h, p - R[:, 2] * h]
    seg = np.clip(lo[2], -h, h)
    if np.sum((lo - [0, 0, seg]) ** 2) <= r * r:
        return np.inf
    best = min(np_sphere(e, r, o, d) for e in ends)   # whole end spheres: inside the capsule where they overlap the cylinder
    a, b, c = ld[0] ** 2 + ld[1] ** 2, lo[0] * ld[0] + lo[1] * ld[1], lo[0] ** 2 + lo[1] ** 2 - r * r
    if a > 1e-15 and b * b - a * c >= 0:
        t = (-b - np.sqrt(b * b - a * c)) / a
        if t > 0 and abs(lo[2] + t * ld[2]) <= h:
            best = min(best, t)
    return best


def np_render(scene, moving, cpos, cR, fovy, W, H, zfar, hf=None):
    org, d, nd = pixel_rays(np.asarray(cpos, float), cR, fovy, W, H)
    depth, geom = np.full(W * H, float(zfar)), np.full(W * H, -1)
    for i in range(W * H):
        st = TR.np_cast(scene, org[i:i + 1], d[i:i + 1], zfar * nd[i], hf)[0]
        best, gb = (st[0], int(st[2])) if st[2] >= 0 and st[0] > 0 else (np.inf, -1)
        for m in range(len(moving.type)):
            t = np_moving(moving.type[m], moving.pos[m], moving.R[m], moving.size[m], org[i], d[i])
            if t <= zfar * nd[i] and t < best:
                best, gb = t, 100 + m
        if gb >= 0:
            depth[i], geom[i] = best / nd[i], gb
    return depth.reshape(H, W), geom.reshape(H, W)


class RandomMoving:
    def __init__(self, rng, n=9):
        self.type = np.array([(2, 3, 6)[i % 3] for i in range(n)], dtype=np.int32)
        self.pos = rng.uniform([-1, -1, 0.2], [1, 1, 1.4], size=(n, 3))
        self.R = np.array([RS.quat2mat(rng.normal(size=4)) for _ in range(n)])
        self.size = np.stack([rng.uniform(0.05, 0.25, n), rng.uniform(0.05, 0.3, n), rng.uniform(0.05, 0.2, n)], 1)


def look_at(eye, target, rng):
    z = np.asarray(eye, float) - target
    z /= np.linalg.norm(z)
    x = np.cross(rng.normal(size=3) * 0.1 + [0, 0, 1], z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1)


@pytest.mark.parametrize('seed', [0, 1, 2, 3])
def test_oracle_vs_numpy_random_scenes(seed):
    rng = np.random.default_rng(100 + seed)
    sim = CS.EmuCam('cassie')
    sc = TR.stairs_scene(sim, rng)
    mv = RandomMoving(rng)
    W, H, zfar = 20, 14, 4.0
    cams = [np.array([2.5, 0.3, 1.2]), np.array([-2.0, -1.5, 0.8])]
    cams.append(mv.pos[0] + RS.quat2mat([1, 0, 0, 0]) @ [0.01, 0.0, 0.0])            # inside a sphere: it is not seen
    cams.append(mv.pos[1] + mv.R[1][:, 2] * (mv.size[1][1] + 0.5 * mv.size[1][0]))    # inside a capsule's cap
    cams.append(mv.pos[2] + 0.5 * mv.R[2] @ mv.size[2])                                 # inside a box
    seen = set()
    for k, eye in enumerate(cams):
        cR = look_at(eye, [0, 0, 0.6], rng)
        a, ga = CS.oracle_render(sc, mv, eye, cR, 60 + 10 * k, W, H, zfar)
        b, gb = np_render(sc, mv, eye, cR, 60 + 10 * k, W, H, zfar)
        assert np.array_equal(ga, gb), np.argwhere(ga != gb)[:5]
        assert np.abs(a - b).max() <= 1e-12
        if k >= 2:
            assert 100 + (k - 2) not in set(ga.ravel())   # the geom the camera sits in
        seen |= set(ga.ravel())
    assert {100, 101, 102} & seen and -1 in seen and any(0 <= g < 100 for g in seen)
    sim.close()


def test_capsule_caps_and_grazes():
    """a capsule seen end-on (the cap only), side-on and at a graze of its silhouette"""
    rng = np.random.default_rng(7)
    sim = CS.EmuCam('cassie')
    sc = sim.scene()

    class M:
        type = np.array([3], dtype=np.int32)
        pos = np.array([[40.0, 0.0, 1.0]])
        R = np.eye(3)[None]
        size = np.array([[0.2, 0.4, 0.0]])
    for eye in ([40.0, 0.0, 3.0], [42.0, 0.0, 1.0], [42.0, 0.2 + 1e-9, 1.0]):
        cR = look_at(eye, M.pos[0], rng)
        a, ga = CS.oracle_render(sc, M, eye, cR, 50, 16, 16, 5.0)
        b, gb = np_render(sc, M, eye, cR, 50, 16, 16, 5.0)
        assert np.array_equal(ga, gb) and np.abs(a - b).max() <= 1e-12
    a, _ = CS.oracle_render(sc, M, [40.0, 0.0, 3.0], np.eye(3), 1.0, 1, 1, 5.0)   # straight down onto the top cap: 3 - 1 - 0.4 - 0.2
    assert abs(a[0, 0] - 1.4) < 1e-12
    sim.close()


# ------------------------------------------------------------------ 2. emulation vs oracle
def states(name, rng):
    """standing, mid-fall and crossed-leg qpos of the fp64 oracle stepper"""
    o = O.OracleSim(os.path.join(G, name + '.omodel'))
    q0 = np.array(o.arr('qpos')).copy()
    qs = [q0.copy()]
    q = o.arr('qpos')
    q[2] += 0.4
    q[3:7] = TR.O_quat_mul(TR.quat_z(rng.uniform(-3, 3)), TR.quat_axis([1, 0.4, 0], 0.5))
    for _ in range(120):
        o.mj_step()
    qs.append(np.array(o.arr('qpos')).copy())
    qc = q0.copy()
    qc[7], qc[21] = -0.3, 0.3    # hip rolls inward: the legs cross in front of a downward camera
    qc[9], qc[23] = 0.6, 0.6
    qs.append(qc)
    o.close()
    return qs


SETUPS = {
    # model: (camera: fixture name or (body, pos, quat, fovy)), zfar
    'cassie_depth': ('egocentric', 4.0),
    'cassie_hfield': ('egocentric', 4.0),
    'cassie': (('cassie-pelvis', [0.3, 0.0, 0.3], TR.quat_axis([0, 1, 0], 0.9), 70.0), 5.0),
    'cassie_tray_box': (('cassie-pelvis', [0.8, 0.0, 0.9], TR.quat_axis([0, 1, 0], 0.8), 60.0), 3.0),
}


def camera_of(model, sim):
    cam, zfar = SETUPS[model]
    if isinstance(cam, str):
        body, pos, quat, fovy, mode = CS.cameras_fixture()[(model, cam)]
        assert mode == 0
    else:
        body, pos, quat, fovy = cam
    return sim.body(body), np.asarray(pos, float), np.asarray(quat, float), fovy, zfar


@pytest.mark.parametrize('fp32', [False, True])
@pytest.mark.parametrize('model', list(SETUPS))
def test_emulation_matches_oracle(model, fp32):
    rng = np.random.default_rng(11)
    sim = CS.EmuCam(model, fp32)
    body, pos, quat, fovy, zfar = camera_of(model, sim)
    W, H = 24, 18
    qs = states(model, rng)
    n = len(qs)
    sc0 = sim.scene()
    scenes, genv, bank = [sc0] * n, None, None
    if model == 'cassie':
        scenes = [TR.stairs_scene(sim, rng) for _ in range(n)]
        for sc, q in zip(scenes, qs):   # stairs in front of the robot, where the camera looks
            for k, g in enumerate(sc.slots):
                if sc.type[k] == 6:
                    sc.pos[k][:2] += q[:2] + [1.2, 0]
        genv = np.array([s.genv_row() for s in scenes])
    if model == 'cassie_hfield':
        bank = np.stack([TR.terrain(rng, sc0) * 0.6 for _ in range(4)])
    out = sim.render(body, pos, quat, fovy, W, H, zfar, n=n, qpos=np.array(qs), genv=genv, bank=bank)
    nmov = 0
    for e in range(n):
        xpos, xquat = CS.oracle_poses(model, qs[e])
        mv = CS.Moving(sim.table, sim.moving_geoms, xpos, xquat)
        cpos, cR = CS.camera_world(xpos, xquat, body, pos, quat / np.linalg.norm(quat))
        hf = None if bank is None else bank[e % 4]
        a, ga = CS.oracle_render(scenes[e], mv, cpos, cR, fovy, W, H, zfar, hf)
        nmov += (ga >= 100).sum()
        assert (ga >= 0).mean() > 0.3
        if not fp32:
            assert np.abs(out[e] - a).max() <= 1e-12, np.abs(out[e] - a).max()
            continue
        amb = CS.ambiguous(scenes[e], mv, cpos, cR, fovy, W, H, zfar, hf)
        assert amb.mean() < 0.005, amb.mean()
        assert np.abs(out[e] - a)[~amb].max() <= 1e-5 * zfar
    if model in ('cassie', 'cassie_tray_box'):
        assert nmov > 0   # the legs, the tray or the cup are in view
    sim.close()


# ------------------------------------------------------------------ 3. body poses
@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_body_poses_match_step_frames(model):
    import test_frames as TF
    rng = np.random.default_rng(3)
    sim = CS.EmuCam(model)
    fs = TF.FrameSim(model)
    names = [b for b in sim.table['names_body'][1:]]
    assert fs.set_frames(names, [0] * len(names)) == 0
    for q in states(model, rng):
        sim.set_qpos(q)
        _, st = sim.render(0, [0, 0, 0], [1, 0, 0, 0], 45, 1, 1, 1.0, poses=True)
        a = RS._d(q)
        fs.L.emu_set(fs.h, b'qpos', a.ctypes.data_as(RS.dp), a.size)
        fs.forward()
        rows = fs.frames()
        for i in range(len(names)):
            b = i + 1
            assert np.abs(st[3 * b:3 * b + 3] - rows[i][0:3]).max() <= 1e-15, names[i]
            assert np.abs(st[96 + 4 * b:96 + 4 * b + 4] - rows[i][3:7]).max() <= 1e-15, names[i]
    fs.close()
    sim.close()


# ------------------------------------------------------------------ 4. known geometry
@pytest.mark.parametrize('fp32', [False, True])
def test_flat_floor_straight_down_and_tilted(fp32):
    sim = CS.EmuCam('cassie_depth', fp32)
    tol = 1e-12 if not fp32 else 2e-6
    for h in (0.5, 1.7):
        d = sim.render(0, [50.0, 0.0, h], [1, 0, 0, 0], 60.0, 32, 24, 5.0)[0]   # on the world body, far from the robot
        assert np.abs(d - h).max() <= tol * 5
    th, h, fovy, W, H = 0.4, 1.2, 50.0, 20, 30
    d = sim.render(0, [50.0, 0.0, h], TR.quat_axis([1, 0, 0], th), fovy, W, H, 10.0)[0]
    ty = np.tan(np.radians(fovy) / 2)
    y = (1 - 2 * (np.arange(H) + 0.5) / H) * ty
    want = h / (np.cos(th) - np.sin(th) * y)
    want = np.where(want > 0, np.minimum(want, 10.0), 10.0)
    assert np.abs(d - want[:, None]).max() <= tol * 10
    sim.close()


# ------------------------------------------------------------------ 5. checks
def test_camera_is_checked():
    sim = CS.EmuCam('cassie')
    ok = dict(body=1, pos=[0, 0, 0], quat=[1, 0, 0, 0], fovy=45, W=8, H=8, zfar=2.0)
    assert sim.render(**ok) is not None
    for bad in (dict(body=99), dict(quat=[0, 0, 0, 0]), dict(quat=[np.nan, 0, 0, 1]), dict(fovy=0), dict(fovy=180), dict(W=257), dict(H=0),
                dict(zfar=0.0), dict(zfar=np.inf)):
        assert sim.render(**{**ok, **bad}) is None, bad
    a = sim.render(**{**ok, 'quat': [2, 0, 0, 0]})   # quaternions are normalised
    assert np.array_equal(a, sim.render(**ok))
    sim.close()
