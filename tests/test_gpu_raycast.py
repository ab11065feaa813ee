"""Terrain ray casting on the H100 (cassie_batch_raycast): the device rows against the fp64 ray oracle (tests/ray_oracle.c) at each sampled
environment's own state, placement and terrain; casting leaves stepping bitwise unchanged; the verbs' semantics and error cases.

Scan: 17 x 11 heading-frame rays at 0.1 m plus 8 root-frame rays.  fp64: distances and hit z within 1e-12, equal geom slots.  fp32: geom slots
equal, distances and hit z within 1e-5 x max on every ray whose hit / miss or slot does not change in the oracle when its origin moves by 1e-5 m in
x or y (edge grazes, fewer than 0.5 % of all sampled rays).  The legacy rangefinders (CassieSim.sense_ground) against the same oracle."""
import os

import numpy as np
import pytest

import oracle as O
import raycast_support as RS
from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, product
from raycast_support import HEADING, ROOT

pytestmark = pytest.mark.gpu

XS, YS = np.arange(-8, 9) * 0.1, np.arange(-5, 6) * 0.1
MAXD = 3.0


def scan_table(rng):
    org_s, d_s = RS.height_scan(XS, YS, 1.0)
    org_r = rng.uniform(-0.2, 0.2, size=(8, 3))
    d_r = rng.normal(size=(8, 3)) * [0.5, 0.5, 0.2] - [0, 0, 1.0]
    d_r /= np.linalg.norm(d_r, axis=1)[:, None]
    kinds = np.array([HEADING] * len(org_s) + [ROOT] * 8)
    return kinds, np.vstack([org_s, org_r]), np.vstack([d_s, d_r])


def slot_scene(name):
    """the model's static geoms in collision-slot order (slot map from the host emulation's build of the same table)"""
    import ctypes as C
    L = RS.emu_lib()
    h = L.emu_new(os.path.join(RS.MODELS, name + '.cmodel').encode(), 0)
    slots = (C.c_int * 16)()
    ns = L.emu_ray_slots(h, slots)
    L.emu_free(h)
    return RS.Scene(name, list(slots)[:ns])


def oracle_env(name, scene, q, kinds, org, d, hf=None):
    o = O.OracleSim(os.path.join(GOLDEN, name + '.omodel'))
    o.arr('qpos')[:] = q[:len(o.arr('qpos'))]
    o.forward()
    pos, R = RS.root_pose(o, scene.t['names_body'].index('cassie-pelvis'))
    o.close()
    ow, dw = np.zeros_like(org), np.zeros_like(d)
    for kind in (HEADING, ROOT):
        m = kinds == kind
        ow[m], dw[m] = RS.world_rays(kind, org[m], d[m], pos, R)
    return RS.oracle_cast(scene, ow, dw, MAXD, hf), ow, dw


def compare(rows, ref, fp32, amb):
    """fp64: equal slots, distance and hit z within 1e-12.  fp32: equal slots, distance and hit z (end-point z for a miss) within 1e-5 x max on
    every ray that is not ambiguous; returns the number of ambiguous rays"""
    if not fp32:
        assert np.array_equal(rows[:, 2], ref[:, 2]), np.nonzero(rows[:, 2] != ref[:, 2])
        assert np.abs(rows[:, :2] - ref[:, :2]).max() <= 1e-12
        return 0
    ok = ~amb
    assert np.array_equal(rows[ok, 2], ref[ok, 2]), np.nonzero((rows[:, 2] != ref[:, 2]) & ok)
    assert np.abs(rows[ok, :2] - ref[ok, :2]).max() <= 1e-5 * MAXD
    return int(amb.sum())


def stepped_batch(P, name, n, prec, ticks, terrains=None):
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
    if ticks:
        b.step(ticks)
    return b


CASES = [('bank', 4096, 'fp32'), ('stairs', 4096, 'fp32'), ('bank', 256, 'fp64'), ('stairs', 256, 'fp64')]


@pytest.mark.parametrize('kind,n,prec', CASES)
def test_scan_matches_oracle(kind, n, prec):
    P = product()
    fp32 = prec == 'fp32'
    rng = np.random.default_rng(11)
    name = 'cassie_hfield' if kind == 'bank' else 'cassie'
    scene0 = slot_scene(name)
    terrains = None
    if kind == 'bank':   # bench.py config 4's kind: 64 terrains, 5 cm of relief, a flat centre patch
        terrains = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
        terrains[:, 95:105, 95:105] = 0
    b = stepped_batch(P, name, n, P.FP32 if fp32 else P.FP64, 300 if kind == 'bank' else 0, terrains)
    scenes = None
    if kind == 'stairs':   # per-environment stairs and floor tilt
        floor = [scene0.t['names_geom'][g] for g in scene0.slots if scene0.type[scene0.slots.index(g)] == 0][0]
        boxes = [scene0.t['names_geom'][g] for g in scene0.slots if scene0.type[scene0.slots.index(g)] == 6][:6]
        q = b.qpos()
        tilt = rng.uniform(0, 0.12, n)
        ax = rng.normal(size=(n, 2))
        ax /= np.linalg.norm(ax, axis=1)[:, None]
        fq = np.stack([np.cos(tilt / 2), ax[:, 0] * np.sin(tilt / 2), ax[:, 1] * np.sin(tilt / 2), np.zeros(n)], 1)
        b.set_env_geom_pose(floor, pos=np.zeros((n, 3)), quat=fq)
        placed = {floor: (np.zeros((n, 3)), fq, None)}
        for j, bx in enumerate(boxes):
            pos = np.column_stack([q[:, 0] + rng.uniform(-1, 1, n), q[:, 1] + rng.uniform(-0.7, 0.7, n), rng.uniform(-0.1, 0.15, n)])
            yaw = rng.uniform(-np.pi, np.pi, n)
            bq = np.stack([np.cos(yaw / 2), np.zeros(n), np.zeros(n), np.sin(yaw / 2)], 1)
            size = rng.uniform([0.1, 0.1, 0.05], [0.5, 0.5, 0.3], size=(n, 3))
            b.set_env_geom_pose(bx, pos=pos, quat=bq, size=size)
            placed[bx] = (pos, bq, size)
        scenes = placed
    kinds, org, d = scan_table(rng)
    b.set_rays(org, d, frame=list(kinds), max_dist=MAXD)
    assert b.nrays() == len(org)
    b.raycast()
    rows, qpos = b.rays(), b.qpos()
    assert rows.shape == (n, len(org), 4)
    n_amb, n_rays = 0, 0
    for e in rng.choice(n, 64, replace=False):
        sc = scene0
        if scenes is not None:
            sc = scene0.copy()
            for gname, (pos, quat, size) in scenes.items():
                sc.place(gname, pos=pos[e], quat=quat[e], size=None if size is None else size[e])
        hf = None if terrains is None else terrains[e % 64]
        ref, ow, dw = oracle_env(name, sc, qpos[e], kinds, org, d, hf)
        n_amb += compare(rows[e], ref, fp32, RS.ambiguous(sc, ow, dw, MAXD, hf) if fp32 else None)
        n_rays += len(org)
        assert (ref[:len(XS) * len(YS), 0] >= 0).all()   # every scan ray sees the terrain
    assert n_amb < 0.005 * n_rays
    b.close()


@pytest.mark.parametrize('prec', ['fp32', 'fp64'])
def test_casting_does_not_change_stepping(prec):
    P = product()
    pr = P.FP32 if prec == 'fp32' else P.FP64
    terrains = (np.random.default_rng(7).uniform(0, 1, (64, 200, 200)) * 0.25).astype(np.float32)
    a, c = (stepped_batch(P, 'cassie_hfield', 512, pr, 0, terrains) for _ in range(2))
    for b in (a, c):
        b.enable_aux()
    a.set_height_scan(XS, YS)
    for t in range(50):
        a.raycast()
        a.step(10)
        c.step(10)
    for f in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
        assert np.array_equal(getattr(a, f)(), getattr(c, f)()), f
    a.close()
    c.close()


def test_verbs_and_errors():
    import ctypes as C
    import torch
    P = product()
    b = P.CassieBatch(64, precision=P.FP32)
    assert b.nrays() == 0
    with pytest.raises(RuntimeError):
        b.raycast()                                   # no table
    b.set_height_scan(XS, YS)
    k = len(XS) * len(YS)
    assert b.nrays() == k and b.L.cassie_batch_row_width(b.h, b'rays') == 4 * k
    with pytest.raises(RuntimeError):
        b.rays()                                      # -1 before the first cast
    with pytest.raises(RuntimeError):
        b.torch_view('rays')                          # no rows yet
    b.L.cassie_batch_get_rays.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
    b.raycast()
    assert b.L.cassie_batch_get_rays(b.h, None) == -1    # NULL output
    r = b.rays()
    z0 = b.qpos()[:, 2]
    assert np.abs(r[:, :, 0] - (1.0 + z0[:, None])).max() < 1e-5 and (r[:, :, 2] == 0).all()
    b.sync()
    hs = b.height_scan()
    assert isinstance(hs, torch.Tensor) and hs.shape == (64, k)
    assert np.array_equal(hs.cpu().numpy().astype(np.float64), r[:, :, 1])
    # bad tables change nothing
    for bad in (dict(frame=[7] * k), dict(direction=[0.0, 0.0, 0.0]), dict(max_dist=0.0), dict(max_dist=-1.0)):
        args = dict(origin=np.zeros((k, 3)), direction=[0.0, 0.0, -1.0], frame=[0] * k, max_dist=1.0)
        args.update(bad)
        with pytest.raises(RuntimeError):
            b.set_rays(**args)
        assert b.nrays() == k
    with pytest.raises(RuntimeError):
        b.set_rays(np.zeros((1025, 3)), [0.0, 0.0, -1.0])
    assert np.array_equal(b.rays(), r)                # the rows of the last cast are still there
    # a miss reads -1, slot -1 and the end point's z
    b.set_rays([[0.0, 0.0, 0.5]], [0.0, 0.0, 1.0], 'heading', 2.0)
    with pytest.raises(RuntimeError):
        b.rays()
    b.raycast()
    m = b.rays()[:, 0]
    assert (m[:, 0] == -1).all() and (m[:, 2] == -1).all() and np.abs(m[:, 1] - (z0 + 2.5)).max() < 1e-5
    b.set_rays([[0.0, 0.0, 0.0]], [0.0, 0.0, -1.0], P.RAY_ROOT, 2.0)   # one frame kind as a constant
    assert b.nrays() == 1
    b.set_rays(np.zeros((0, 3)), [0.0, 0.0, -1.0])  # k = 0 drops the table
    assert b.nrays() == 0 and b.L.cassie_batch_row_width(b.h, b'rays') == 0
    with pytest.raises(RuntimeError):
        b.raycast()
    b.close()


def test_sense_ground_matches_oracle_from_the_mirror_site_poses():
    """cassie_no_grav.xml's six rangefinders over a float-down trajectory (no gravity: the pelvis, turned so that the rangefinder sites look down,
    drifts towards the floor at 1 m/s): each reading is the oracle's cast from the site pose the simulator's mirrors hold, along the site's z axis,
    capped at the sensor's cutoff (min(cutoff, d); -1 stays -1)"""
    P = product()
    rf = [ln.split() for ln in open(os.path.join(GOLDEN, 'cassie_no_grav_rangefinders.txt')) if not ln.startswith('#')]
    sites, cut = [x[1] for x in rf], np.array([float(x[2]) for x in rf])
    scene = slot_scene('cassie_no_grav')
    sim = P.CassieSim(P.model_path('cassie_no_grav'))
    q = sim.qpos()
    q[2] = 0.9
    q[3:7] = [0, 1, 0, 0]   # rolled over: the sites' z axes, which point up and back on an upright pelvis, look down and forward
    sim.set_qpos(q)
    v = np.zeros(sim.nv)
    v[2] = -1.0
    sim.set_qvel(v)
    u = P.pd_in_t()
    seen = []
    for t in range(60):
        sim.step_pd(u)
        got = sim.sense_ground()
        org = np.array([sim.get_site_xpos(s) for s in sites])
        dirs = np.array([RS.quat2mat(sim.get_site_quat(s))[:, 2] for s in sites])
        ref = RS.oracle_cast(scene, org, dirs, 1e6)[:, 0]
        want = np.where((cut > 0) & (ref >= 0), np.minimum(cut, ref), ref)
        assert np.abs(got - want).max() <= 1e-12, (t, got, want)
        seen.append(got)
        for _ in range(9):
            sim.step_pd(u)
    seen = np.array(seen)
    assert (seen == 1.0).any() and ((seen >= 0) & (seen < 1.0)).any()   # both capped and measured readings occur
    other = P.CassieSim(P.model_path('cassie'))
    assert np.array_equal(other.sense_ground(), np.zeros(6))               # no rangefinders: zeros and a recorded error
    assert 'rangefinder' in P._last_error()
