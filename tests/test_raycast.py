"""Terrain ray casting on the CPU (DESIGN.md section 3, "Terrain rays").

1. The fp64 ray oracle (tests/ray_oracle.c) against an independent numpy statement of the same rules: Moller-Trumbore over every triangle of the
   cells the ray's xy segment crosses, a slab test for boxes and the plane formula, on cassie.xml with seeded stairs and tilted floors and on
   cassie_hfield.xml with random terrains: distances within 1e-12, equal geom slots.
2. Invariants of the heading-frame height scan, through the oracle and the product's ray source run in the host emulation.
3. The ray source compiled with -DCASSIE_EMU (tests/emu/emu_raycast.cpp) against the oracle: the three frame kinds, with and without per-environment
   static-geom rows, a bank of 4 terrains, fp64 (1e-12) and fp32 (1e-5 of max, ambiguous edge grazes excluded).
"""
import ctypes as C
import os

import numpy as np
import pytest

import oracle as O
import raycast_support as RS
from raycast_support import HEADING, ROOT, WORLD

G = RS.GOLDEN


def quat_z(yaw):
    return [np.cos(yaw / 2), 0, 0, np.sin(yaw / 2)]


def quat_axis(axis, ang):
    a = np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis)
    return np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * a])


class EmuRay:
    """one emulated simulator with the ray source"""

    def __init__(self, name, fp32=False):
        self.L = RS.emu_lib()
        self.h = self.L.emu_new(os.path.join(RS.MODELS, name + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h
        self.name = name
        slots = (C.c_int * 16)()
        self.ns = self.L.emu_ray_slots(self.h, slots)
        self.slots = list(slots)[:self.ns]

    def close(self):
        if self.h:
            self.L.emu_free(self.h)
            self.h = None

    def scene(self):
        return RS.Scene(self.name, self.slots)

    def set_qpos(self, q):
        a = RS._d(q)
        self.L.emu_set(self.h, b'qpos', a.ctypes.data_as(RS.dp), a.size)
        self.L.emu_forward(self.h)

    def set_hfield(self, data):
        a = np.ascontiguousarray(data, dtype=np.float32).ravel()
        self.L.emu_set_hfield(self.h, a.ctypes.data_as(C.POINTER(C.c_float)), a.size)

    def root(self):
        out = np.zeros(12)
        self.L.emu_ray_root(self.h, out.ctypes.data_as(RS.dp))
        return out[:3], out[3:].reshape(3, 3)

    def cast(self, kinds, org, dirs, maxd, n=1, qpos=None, genv=None, bank=None):
        k = len(org)
        out = np.zeros((n, k, 4))
        fr = (C.c_int * k)(*[int(x) for x in np.broadcast_to(kinds, (k,))])
        o, d, m = RS._d(org), RS._d(dirs), RS._d(np.broadcast_to(maxd, (k,)))
        q = None if qpos is None else RS._d(qpos)
        g = None if genv is None else RS._d(genv)
        b = None if bank is None else np.ascontiguousarray(bank, dtype=np.float32)
        rc = self.L.emu_ray_cast(self.h, n, None if q is None else q.ctypes.data_as(RS.dp), 0 if q is None else q.shape[1],
                                 None if g is None else g.ctypes.data_as(RS.dp), None if b is None else b.ctypes.data_as(C.POINTER(C.c_float)),
                                 0 if b is None else len(b), fr, o.ctypes.data_as(RS.dp), d.ctypes.data_as(RS.dp), m.ctypes.data_as(RS.dp), k,
                                 out.ctypes.data_as(RS.dp))
        assert rc == 0
        return out


# ------------------------------------------------------------------ the independent numpy statement
def np_cast(scene, org, dirs, maxd, hf=None):
    out = np.zeros((len(org), 4))
    for i, (o, d) in enumerate(zip(org, dirs)):
        best, gb = -1.0, -1
        for g, ty in enumerate(scene.type):
            p, R, s = scene.pos[g], scene.R[g], scene.size[g]
            lo, ld = R.T @ (o - p), R.T @ d
            t = -1.0
            if ty == 0:   # plane: z = 0 of its frame, front face, inside the rectangle
                if ld[2] < -1e-15:
                    t = -lo[2] / ld[2]
                    x = lo + t * ld
                    if t < 0 or (s[0] > 0 and abs(x[0]) > s[0]) or (s[1] > 0 and abs(x[1]) > s[1]):
                        t = -1.0
            elif ty == 6:   # box: slabs
                with np.errstate(divide='ignore', invalid='ignore'):
                    a, b = (-s - lo) / ld, (s - lo) / ld
                par = ld == 0
                if np.any(par & (np.abs(lo) > s)):
                    t = -1.0
                else:
                    t0 = np.max(np.where(par, -np.inf, np.minimum(a, b)))
                    t1 = np.min(np.where(par, np.inf, np.maximum(a, b)))
                    t = -1.0 if (t1 < t0 or t1 < 0) else (t0 if t0 >= 0 else t1)
            elif ty == 1 and hf is not None:
                t = np_hfield(scene, hf, o - p, d, maxd)
            if 0 <= t <= maxd and (gb < 0 or t < best):
                best, gb = t, g
        out[i] = [best if gb >= 0 else -1, o[2] + (best if gb >= 0 else maxd) * d[2], gb, 0]
    return out


def np_hfield(scene, hf, o, d, maxd):
    sx, sy, sz = scene.hsize[:3]
    nrow, ncol = scene.nrow, scene.ncol
    dx, dy = 2 * sx / (ncol - 1), 2 * sy / (nrow - 1)
    ts = np.array([0.0, maxd])
    for ax, h in ((0, sx), (1, sy)):   # the segment clipped to the field
        if d[ax] == 0:
            if abs(o[ax]) > h:
                return -1.0
            continue
        a, b = sorted([(-h - o[ax]) / d[ax], (h - o[ax]) / d[ax]])
        ts = np.array([max(ts[0], a), min(ts[1], b)])
    if ts[0] > ts[1]:
        return -1.0
    x, y = o[0] + ts * d[0], o[1] + ts * d[1]
    cs = np.arange(max(0, int(np.floor((x.min() + sx) / dx)) - 1), min(ncol - 2, int(np.floor((x.max() + sx) / dx)) + 1) + 1)
    rs = np.arange(max(0, int(np.floor((y.min() + sy) / dy)) - 1), min(nrow - 2, int(np.floor((y.max() + sy) / dy)) + 1) + 1)
    if not len(cs) or not len(rs):
        return -1.0
    C_, R_ = np.meshgrid(cs, rs)
    C_, R_ = C_.ravel(), R_.ravel()
    x0, y0 = -sx + C_ * dx, -sy + R_ * dy
    z = lambda r, c: hf[r, c].astype(np.float64) * sz   # noqa: E731
    v00 = np.stack([x0, y0, z(R_, C_)], 1)
    v10 = np.stack([x0 + dx, y0, z(R_, C_ + 1)], 1)
    v01 = np.stack([x0, y0 + dy, z(R_ + 1, C_)], 1)
    v11 = np.stack([x0 + dx, y0 + dy, z(R_ + 1, C_ + 1)], 1)
    best = -1.0
    for a, b, c in ((v00, v10, v01), (v10, v11, v01)):   # Moller-Trumbore over every triangle, both faces
        e1, e2 = b - a, c - a
        p = np.cross(d, e2)
        det = np.einsum('ij,ij->i', e1, p)
        ok = np.abs(det) >= 1e-15
        det = np.where(ok, det, 1.0)
        sv = o - a
        u = np.einsum('ij,ij->i', sv, p) / det
        q = np.cross(sv, e1)
        v = (q @ d) / det
        t = np.einsum('ij,ij->i', e2, q) / det
        eps = 1e-12
        hit = ok & (u >= -eps) & (u <= 1 + eps) & (v >= -eps) & (u + v <= 1 + eps) & (t >= ts[0]) & (t <= ts[1])
        if hit.any():
            tm = t[hit].min()
            best = tm if best < 0 else min(best, tm)
    return best


# ------------------------------------------------------------------ scenes
def stairs_scene(sim, rng, n_boxes=6):
    sc = sim.scene()
    boxes = [sc.t['names_geom'][g] for g in sc.slots if int(sc.t['geom_type'][g]) == 6]
    for j, name in enumerate(boxes[:n_boxes]):
        sc.place(name, pos=[rng.uniform(-1, 1.5), rng.uniform(-1, 1), rng.uniform(-0.1, 0.2)], quat=quat_z(rng.uniform(-np.pi, np.pi)),
                 size=[rng.uniform(0.1, 0.5), rng.uniform(0.1, 0.5), rng.uniform(0.05, 0.3)])
    floor = [sc.t['names_geom'][g] for g in sc.slots if int(sc.t['geom_type'][g]) == 0][0]
    sc.place(floor, pos=[0, 0, rng.uniform(-0.1, 0.1)], quat=quat_axis([rng.normal(), rng.normal(), 0], rng.uniform(0, 0.15)))
    return sc


def random_rays(rng, k, centre=(0, 0, 1.0)):
    org = np.asarray(centre) + rng.uniform(-1.5, 1.5, size=(k, 3)) * [1, 1, 0.4]
    d = rng.normal(size=(k, 3)) * [1, 1, 0.5] - [0, 0, 1.0]
    d[: k // 4] = [0, 0, -1.0]   # a quarter vertical (the height-field fast path)
    return org, d / np.linalg.norm(d, axis=1)[:, None]


def terrain(rng, sc):
    return rng.uniform(0, 1, size=(sc.nrow, sc.ncol)).astype(np.float32)


# ------------------------------------------------------------------ 1. oracle vs numpy
@pytest.mark.parametrize('seed', [0, 1, 2])
def test_oracle_vs_numpy_stairs_and_tilt(seed):
    rng = np.random.default_rng(seed)
    sim = EmuRay('cassie')
    sc = stairs_scene(sim, rng)
    org, d = random_rays(rng, 400)
    a, b = RS.oracle_cast(sc, org, d, 3.0), np_cast(sc, org, d, 3.0)
    assert np.array_equal(a[:, 2], b[:, 2])
    assert np.abs(a[:, :2] - b[:, :2]).max() <= 1e-12
    assert (a[:, 0] >= 0).mean() > 0.5 and len(set(a[:, 2])) > 3   # the rays meet the floor and several boxes
    sim.close()


@pytest.mark.parametrize('seed', [0, 1])
def test_oracle_vs_numpy_hfield(seed):
    rng = np.random.default_rng(10 + seed)
    sim = EmuRay('cassie_hfield')
    sc = sim.scene()
    hf = terrain(rng, sc)
    org, d = random_rays(rng, 300, centre=(0, 0, 0.6))
    a, b = RS.oracle_cast(sc, org, d, 3.0, hf), np_cast(sc, org, d, 3.0, hf)
    assert np.array_equal(a[:, 2], b[:, 2])
    assert np.abs(a[:, :2] - b[:, :2]).max() <= 1e-12
    assert (a[:, 2] == sc.type.tolist().index(1)).mean() > 0.5
    sim.close()


# ------------------------------------------------------------------ 2. invariants
def standing_qpos(name, z=1.0, yaw=0.0, tilt=0.0):
    o = O.OracleSim(os.path.join(G, name + '.omodel'))
    q = np.array(o.arr('qpos')).copy()
    q[2] = z
    rq = O_quat_mul(quat_z(yaw), quat_axis([1, 0.3, 0], tilt))
    q[3:7] = rq
    o.close()
    return q


def O_quat_mul(a, b):
    w1, x1, y1, z1 = a
    w2, x2, y2, z2 = b
    return np.array([w1*w2 - x1*x2 - y1*y2 - z1*z2, w1*x2 + x1*w2 + y1*z2 - z1*y2, w1*y2 - x1*z2 + y1*w2 + z1*x2, w1*z2 + x1*y2 - y1*x2 + z1*w2])


def test_flat_floor_scan_reads_height_and_box_reads_less():
    sim = EmuRay('cassie')
    q = standing_qpos('cassie', z=1.0, yaw=0.7, tilt=0.2)
    sim.set_qpos(q)
    pos, R = sim.root()
    org, d = RS.height_scan(np.arange(-8, 9) * 0.1, np.arange(-5, 6) * 0.1, 1.0)
    r = sim.cast(HEADING, org, d, 3.0)[0]
    assert np.all(r[:, 2] == 0) and np.abs(r[:, 0] - (1.0 + pos[2])).max() < 1e-12 and np.abs(r[:, 1]).max() < 1e-12
    # a box of height h under the pattern
    sc = sim.scene()
    name = sc.t['names_geom'][[g for g in sc.slots if int(sc.t['geom_type'][g]) == 6][0]]
    h = 0.25
    k = sc.place(name, pos=[pos[0], pos[1], h / 2], quat=[1, 0, 0, 0], size=[2, 2, h / 2])
    r2 = sim.cast(HEADING, org, d, 3.0, genv=sc.genv_row()[None])[0]
    assert np.all(r2[:, 2] == k) and np.abs(r2[:, 0] - (1.0 + pos[2] - h)).max() < 1e-12
    sim.close()


def test_heading_frame_turns_with_yaw_not_with_pitch_roll():
    """an off-axis box under part of a 21 x 21 scan: which rays read the box follows the root's yaw (a quarter turn moves the hits to the rays
    the turned pattern puts over the box), and pitch / roll of the root change nothing"""
    sim = EmuRay('cassie')
    sc = sim.scene()
    name = sc.t['names_geom'][[g for g in sc.slots if int(sc.t['geom_type'][g]) == 6][0]]
    h = 0.3
    k = sc.place(name, pos=[0.0, 0.8, h / 2], quat=[1, 0, 0, 0], size=[0.25, 0.25, h / 2])
    g = np.arange(-10, 11) * 0.1
    org, d = RS.height_scan(g, g, 1.0)
    hits = {}
    for yaw, pitch, roll in ((0.0, 0.0, 0.0), (np.pi / 2, 0.0, 0.0), (np.pi / 2, 0.3, -0.2)):
        q = standing_qpos('cassie', 1.0)
        q[0:2] = 0
        q[3:7] = O_quat_mul(O_quat_mul(quat_z(yaw), quat_axis([0, 1, 0], pitch)), quat_axis([1, 0, 0], roll))
        sim.set_qpos(q)
        pos, R = sim.root()
        r = sim.cast(HEADING, org, d, 3.0, genv=sc.genv_row()[None])[0]
        c, s_ = np.cos(yaw), np.sin(yaw)
        w = org[:, :2] @ np.array([[c, -s_], [s_, c]]).T   # where the heading frame puts each ray
        want = (np.abs(w[:, 0]) < 0.25) & (np.abs(w[:, 1] - 0.8) < 0.25)
        assert np.array_equal(r[:, 2] == k, want)
        assert np.abs(r[want, 0] - (1.0 + pos[2] - h)).max() < 1e-12 and np.abs(r[~want, 0] - (1.0 + pos[2])).max() < 1e-12
        hits[(yaw, pitch, roll)] = r
    assert want.sum() == 25 and not np.array_equal(hits[(0.0, 0.0, 0.0)][:, 2], hits[(np.pi / 2, 0.0, 0.0)][:, 2])
    assert np.array_equal(hits[(np.pi / 2, 0.0, 0.0)], hits[(np.pi / 2, 0.3, -0.2)])
    sim.close()


def test_front_face_and_floor_extent():
    sim = EmuRay('cassie')
    sc = sim.scene()
    org = np.array([[0, 0, -0.5], [0, 0, -0.5], [0, 9.9, 1], [0, 10.1, 1], [0, -10.1, 1], [0, 0, 1]])
    d = np.array([[0, 0, -1], [0, 0, 1], [0, 0, -1], [0, 0, -1], [0, 0, -1], [0, 0, -1.0]])
    a = RS.oracle_cast(sc, org, d, 3.0)
    e = sim.cast(WORLD, org, d, 3.0)[0]
    assert np.array_equal(a[:, 2], e[:, 2]) and np.abs(a[:, :2] - e[:, :2]).max() < 1e-12
    assert list(a[:, 0] >= 0) == [False, False, True, False, False, True]   # below the floor: no hit either way; |y| > 10: off the floor
    sim.close()


# ------------------------------------------------------------------ 3. emulation vs oracle
def oracle_rows(sim, scene, q, kinds, org, d, maxd, hf=None):
    """the oracle's rows for one environment at qpos q: root pose from the oracle stepper's kinematics"""
    o = O.OracleSim(os.path.join(G, sim.name + '.omodel'))
    o.arr('qpos')[:] = q[:len(o.arr('qpos'))]
    o.forward()
    pos, R = RS.root_pose(o, scene.t['names_body'].index('cassie-pelvis'))
    o.close()
    ow, dw = np.zeros_like(org), np.zeros_like(d)
    for kind in (HEADING, ROOT, WORLD):
        m = np.asarray(kinds) == kind
        if m.any():
            ow[m], dw[m] = RS.world_rays(kind, org[m], d[m], pos, R)
    return RS.oracle_cast(scene, ow, dw, maxd, hf), (ow, dw)


def mixed_rays(rng):
    org_s, d_s = RS.height_scan(np.arange(-8, 9) * 0.1, np.arange(-5, 6) * 0.1, 1.0)
    org_r = rng.uniform(-0.3, 0.3, size=(8, 3))
    d_r = rng.normal(size=(8, 3)) - [0, 0, 2.0]
    org_w, d_w = random_rays(rng, 24)
    kinds = [HEADING] * len(org_s) + [ROOT] * 8 + [WORLD] * 24
    return np.array(kinds), np.vstack([org_s, org_r, org_w]), np.vstack([d_s, d_r / np.linalg.norm(d_r, axis=1)[:, None], d_w])


def check(e, a, fp32, amb, maxd):
    if not fp32:
        assert np.array_equal(e[:, 2], a[:, 2]), np.nonzero(e[:, 2] != a[:, 2])
        assert np.abs(e[:, :2] - a[:, :2]).max() <= 1e-12
        return
    assert amb.mean() < 0.005
    ok = ~amb
    assert np.array_equal(e[ok, 2], a[ok, 2])
    hit = ok & (a[:, 0] >= 0)
    assert np.abs(e[hit, 0] - a[hit, 0]).max() <= 1e-5 * maxd
    assert np.abs(e[ok, 1] - a[ok, 1]).max() <= 1e-5 * maxd   # hit z, or the end point's z for a miss


@pytest.mark.parametrize('fp32', [False, True])
def test_emulation_matches_oracle_stairs(fp32):
    rng = np.random.default_rng(5)
    sim = EmuRay('cassie', fp32)
    n = 4
    qs, scenes, rows = [], [], []
    for e in range(n):
        q = standing_qpos('cassie', rng.uniform(0.8, 1.1), rng.uniform(-3, 3), rng.uniform(0, 0.3))
        q[0:2] = rng.uniform(-0.5, 0.5, 2)
        qs.append(q)
        sc = stairs_scene(sim, rng)
        scenes.append(sc)
        rows.append(sc.genv_row())
    kinds, org, d = mixed_rays(rng)
    out = sim.cast(kinds, org, d, 3.0, n=n, qpos=np.array(qs), genv=np.array(rows))
    plain = sim.cast(kinds, org, d, 3.0, n=1, qpos=np.array(qs[:1]))[0]   # without rows: the model block's placement
    for e in range(n):
        a, (ow, dw) = oracle_rows(sim, scenes[e], qs[e], kinds, org, d, 3.0)
        amb = RS.ambiguous(scenes[e], ow, dw, 3.0) if fp32 else None
        check(out[e], a, fp32, amb, 3.0)
    a0, (ow, dw) = oracle_rows(sim, sim.scene(), qs[0], kinds, org, d, 3.0)
    check(plain, a0, fp32, RS.ambiguous(sim.scene(), ow, dw, 3.0) if fp32 else None, 3.0)
    sim.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_emulation_matches_oracle_terrain_bank(fp32):
    rng = np.random.default_rng(7)
    sim = EmuRay('cassie_hfield', fp32)
    sc = sim.scene()
    K, n = 4, 6
    bank = np.stack([terrain(rng, sc) for _ in range(K)])
    qs = []
    for e in range(n):
        q = standing_qpos('cassie_hfield', rng.uniform(0.9, 1.2), rng.uniform(-3, 3), rng.uniform(0, 0.3))
        q[0:2] = rng.uniform(-2, 2, 2)
        qs.append(q)
    kinds, org, d = mixed_rays(rng)
    out = sim.cast(kinds, org, d, 3.0, n=n, qpos=np.array(qs), bank=bank)
    for e in range(n):
        a, (ow, dw) = oracle_rows(sim, sc, qs[e], kinds, org, d, 3.0, bank[e % K])
        amb = RS.ambiguous(sc, ow, dw, 3.0, bank[e % K]) if fp32 else None
        check(out[e], a, fp32, amb, 3.0)
        assert (a[:, 2] == sc.type.tolist().index(1)).mean() > 0.5
    sim.close()


def test_root_pose_matches_pelvis_frame():
    """the root pose the ray source composes equals the pelvis pose of the emulation's kinematics after a forward pass (fp64)"""
    import test_frames as TF
    rng = np.random.default_rng(3)
    sim = EmuRay('cassie')
    fs = TF.FrameSim('cassie')
    assert fs.set_frames(['cassie-pelvis'], [0]) == 0
    for _ in range(4):
        q = standing_qpos('cassie', rng.uniform(0.8, 1.1), rng.uniform(-3, 3), rng.uniform(0, 0.5))
        q[0:2] = rng.uniform(-1, 1, 2)
        sim.set_qpos(q)
        pos, R = sim.root()
        a = RS._d(q)
        fs.L.emu_set(fs.h, b'qpos', a.ctypes.data_as(RS.dp), a.size)
        fs.forward()
        row = fs.frames()[0]
        assert np.abs(pos - row[0:3]).max() <= 1e-15
        assert np.abs(R - RS.quat2mat(row[3:7])).max() <= 1e-15
    fs.close()
    sim.close()


def test_table_is_checked_as_a_whole():
    sim = EmuRay('cassie')
    org, d = np.zeros((2, 3)), np.array([[0, 0, -1.0], [0, 0, -1.0]])
    L = sim.L
    out = np.zeros((1, 2, 4))

    def cast(kinds, dd, mm):
        fr = (C.c_int * 2)(*kinds)
        return L.emu_ray_cast(sim.h, 1, None, 0, None, None, 0, fr, RS._d(org).ctypes.data_as(RS.dp), RS._d(dd).ctypes.data_as(RS.dp),
                              RS._d(mm).ctypes.data_as(RS.dp), 2, out.ctypes.data_as(RS.dp))
    assert cast([0, 2], d, [1.0, 1.0]) == 0
    assert cast([0, 3], d, [1.0, 1.0]) == -1
    assert cast([0, 1], np.array([[0, 0, 0], [0, 0, -1.0]]), [1.0, 1.0]) == -1
    assert cast([0, 1], d, [1.0, 0.0]) == -1
    sim.close()
