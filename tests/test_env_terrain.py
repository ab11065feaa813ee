"""Per-environment terrain (cassie_batch_set_env_hfield): the product's stepper, ray and camera sources in the host emulation, with each environment's
bank entry, height-field position and size taken from its rows (the F_TR instances) instead of e % K and the model block.  The GPU twins are in
tests/test_gpu_env_terrain.py.

The emulation is tests/emu/emu_env_terrain.cpp, built into its own library here.  The fp64 oracle gets an environment's size and the model compiler's
bounding radius for it through a temporary copy of its model table, its position through the live geom_pos array, its terrain through the live
elevation array."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

import raycast_support as RS
from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
CMODEL = os.path.join(MODELS, 'cassie_hfield.cmodel')
OMODEL = os.path.join(GOLDEN, 'cassie_hfield.omodel')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
FALL_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), 0.05 * np.asarray(PD_PGAIN), 0.05 * np.asarray(PD_DGAIN)])   # too weak to hold the robot: it folds and falls
SHARED_SIZE = np.array([5.0, 5.0, 0.2, 0.1])
SHARED_POS = np.array([0.0, 0.0, -0.1])
HF_GEOM = 0   # 'hfield1', in the reference's geom numbering
# four terrains and four placements: elevation scales 0, 0.5x, 1x, 2x, other half-extents, offset positions
SCALES = (0.0, 0.5, 1.0, 2.0)
HALF = ((5.0, 5.0), (4.0, 6.0), (6.5, 3.5), (3.0, 4.5))
OFFSETS = ((0.0, 0.0, 0.0), (0.04, -0.03, 0.02), (-0.05, 0.02, -0.03), (0.02, 0.05, 0.01))

_LIB = None


def terrain_bank(K, seed):
    """K terrains of normalised elevations: rough everywhere (up to 1 cm under the feet at scale 1), rougher away from the centre"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0, 1, (K, 200, 200)).astype(np.float32)
    d[:, 90:110, 90:110] *= 0.05
    return d


def placement(i, base=SHARED_SIZE):
    """the i-th test placement: (pos [3], size [4])"""
    sx, sy = HALF[i % 4]
    return SHARED_POS + np.array(OFFSETS[i % 4]), np.array([sx, sy, SCALES[i % 4] * base[2], base[3]])


def rbound(size):
    """the model compiler's bounding radius of a height field of this size (mjcf.cpp)"""
    return float(np.linalg.norm([size[0], size[1], max(size[2], size[3])]))


def oracle_on(O, data, pos, size):
    """an fp64 oracle of cassie_hfield.xml standing on `data` with the height field at pos / size"""
    lines = open(OMODEL).read().split('\n')
    for i, ln in enumerate(lines):
        t = ln.split()
        if ln.startswith('hfield_size '):
            lines[i] = ' '.join(t[:3] + [repr(float(x)) for x in size])
        elif ln.startswith('geom_rbound '):
            t[3 + HF_GEOM] = repr(rbound(size))
            lines[i] = ' '.join(t)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, 'cassie_hfield.omodel')
        with open(p, 'w') as f:
            f.write('\n'.join(lines))
        o = O.OracleSim(p)
    o.model_arr('geom_pos').reshape(-1, 3)[HF_GEOM] = pos
    a = np.ascontiguousarray(data, dtype=np.float32)
    C.memmove(o.L.osim_hfield_data(o.h), a.ctypes.data, a.nbytes)
    o.forward()
    return o


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_env_terrain.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_env_terrain.cpp', 'emu_camera.cpp', 'emu_raycast.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'raycast.inl', 'camera.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci, ip = C.c_void_p, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int)
        L.emu_tr_new.restype = vp
        L.emu_tr_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_tr_free', 'emu_tr_forward', 'emu_plain'):
            getattr(L, n).argtypes = [vp]
        L.emu_tr_bank.argtypes = [vp, C.POINTER(C.c_float), ci]
        L.emu_tr_set.argtypes = [vp, ci, ci, ci, dp, dp]
        L.emu_tr_step.argtypes = [vp, dp, ci]
        L.emu_tr_row.argtypes = [vp, dp, dp, dp]
        L.emu_tr_ray_cast.argtypes = [vp, ci, dp, ci, dp, ip, ip, dp, dp, dp, ci, dp]
        L.emu_tr_render.argtypes = [vp, ci, dp, ci, dp, ip, ci, dp, dp, C.c_double, ci, ci, C.c_double, dp]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


class TerrainSim:
    """one emulated environment `env` of a batch whose bank is `bank`; mode 0 plain, 1 the F_EG row, 2 per-environment terrain"""

    def __init__(self, bank, fp32=False, plain=True):
        self.L = lib()
        self.h = self.L.emu_tr_new(CMODEL.encode(), 1 if fp32 else 0)
        assert self.h
        if plain:
            self.L.emu_plain(self.h)
        self.bank = np.ascontiguousarray(bank, dtype=np.float32)
        self.L.emu_tr_bank(self.h, self.bank.ctypes.data_as(C.POINTER(C.c_float)), len(self.bank))

    def close(self):
        if self.h:
            self.L.emu_tr_free(self.h)
            self.h = None

    def set(self, mode, env, terrain=0, pos=None, size=None):
        return self.L.emu_tr_set(self.h, mode, env, terrain, _dp(pos), _dp(size))

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def step(self, pd50, nticks=1):
        self.L.emu_tr_step(self.h, _dp(pd50), nticks)

    def forward(self):
        self.L.emu_tr_forward(self.h)

    def row(self, pos=None, size=None):
        out = np.zeros(256)
        self.L.emu_tr_row(self.h, _dp(pos), _dp(size), out.ctypes.data_as(C.POINTER(C.c_double)))
        return out


def hf_scene(sc0, pos, size):
    """the ray / camera oracles' static scene with the height field at pos (in its body frame) and size"""
    sc = sc0.copy()
    k = sc.slot('hfield1')
    b = int(sc.t['geom_bodyid'][HF_GEOM])
    Rb, pb = (np.eye(3), np.zeros(3)) if b == 0 else (RS.quat2mat(sc.t['body_quat'][4 * b:4 * b + 4]), sc.t['body_pos'][3 * b:3 * b + 3])
    sc.pos[k] = pb + Rb @ np.asarray(pos, float)
    sc.hsize = np.ascontiguousarray(size, dtype=np.float64)
    return sc


# ------------------------------------------------------------------ 1. the default row is the F_EG source's result, bitwise
@pytest.mark.parametrize('fp32', [False, True])
def test_default_selection_is_bitwise_the_env_geom_source(fp32):
    """selection e % K with the shared position and size through the F_TR source: bitwise the F_EG source's result (and that of the plain source)"""
    bank = terrain_bank(4, 3)
    sims = [TerrainSim(bank, fp32) for _ in range(3)]
    env = 5
    assert sims[0].set(0, env) == 0 and sims[1].set(1, env) == 0 and sims[2].set(2, env, terrain=env % 4, pos=SHARED_POS, size=SHARED_SIZE) == 0
    sims[0].L.emu_set_hfield.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]   # the plain source stands on the simulator's own terrain
    sims[0].L.emu_set_hfield(sims[0].h, bank[env % 4].ctypes.data_as(C.POINTER(C.c_float)), bank[env % 4].size)
    for s in sims:
        s.forward()
    for k in range(600):
        pd = PD_ROW if k < 300 else FALL_ROW
        for s in sims:
            s.step(pd)
        for f in ('qpos', 'qvel', 'obs', 'counters'):
            a, b, c = (s.get(f) for s in sims)
            assert np.array_equal(b, c) and np.array_equal(a, c), (k, f)
    for s in sims:
        s.close()


# ------------------------------------------------------------------ 2. against the oracle
@pytest.mark.parametrize('case', range(4))
def test_env_terrain_follows_the_oracle(oracle_mod, case):
    """terrain `case` of a 4-terrain bank at elevation scale 0, 0.5x, 1x or 2x, with other half-extents and an offset position; a stance, then the PD
    gains drop and the robot falls onto the terrain.  fp64: qpos within 1e-9 and the same PGS iteration count every tick; fp32: within 1e-3 (the worst-environment bar of DESIGN.md section 3) while
    standing, and the fall stays within 1e-2 (contact make / break amplifies the single-precision round-off)"""
    bank = terrain_bank(4, 17)
    pos, size = placement(case)
    env, t = 6, (case + 1) % 4   # not env % K: the selection decides
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    uf = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=FALL_ROW[30:40], dGain=FALL_ROW[40:50])
    for fp32 in (False, True):
        o = oracle_on(oracle_mod, bank[t], pos, size)
        e = TerrainSim(bank, fp32)
        assert e.set(2, env, terrain=t, pos=pos, size=size) == 0
        e.forward()
        stance, fall, iters_equal, ncon = 0.0, 0.0, True, 0
        for k in range(800):
            fallen = k >= 400
            o.step_pd(uf if fallen else u)
            e.step(FALL_ROW if fallen else PD_ROW)
            d = np.abs(e.get('qpos')[:35] - o.arr('qpos')).max()
            if fallen:
                fall = max(fall, d)
            else:
                stance = max(stance, d)
            iters_equal = iters_equal and int(e.get('counters')[3]) == o.get_int('solver_iter')
            ncon += o.get_int('ncon')
        assert int(e.get('counters')[4]) == 0
        assert ncon > 400, ncon   # on the terrain
        if fp32:
            assert stance < 1e-3 and fall < 1e-2, (case, stance, fall)
        else:
            assert stance < 1e-9 and fall < 1e-9 and iters_equal, (case, stance, fall, iters_equal)
        assert o.arr('qpos')[2] < 0.8   # it fell
        e.close()
        o.close()


def test_selection_and_size_change_the_trajectory():
    """the selection and the size are really read: another terrain, another scale or another position gives another trajectory"""
    bank = terrain_bank(4, 5)
    pos, size = placement(3)
    ref = TerrainSim(bank)
    ref.set(2, 0, terrain=1, pos=pos, size=size)
    others = []
    for t, p, s in ((2, pos, size), (1, pos + [0.05, 0, 0], size), (1, pos, size * [1, 1, 0.5, 1])):
        e = TerrainSim(bank)
        e.set(2, 0, terrain=t, pos=p, size=s)
        others.append(e)
    for s in [ref] + others:
        s.forward()
    for _ in range(300):
        for s in [ref] + others:
            s.step(PD_ROW)
    q = ref.get('qpos')
    for e in others:
        assert np.abs(e.get('qpos') - q).max() > 1e-5


def test_selection_is_read_mod_k():
    """a selection past the bank reads entry t % K: no value addresses outside the bank"""
    bank = terrain_bank(3, 9)
    a, b = TerrainSim(bank), TerrainSim(bank)
    a.set(2, 0, terrain=2)
    b.set(2, 0, terrain=2 + 3 * 7)
    for s in (a, b):
        s.forward()
        s.step(PD_ROW, 200)
    assert np.array_equal(a.get('qpos'), b.get('qpos'))


def test_slot_holds_position_size_and_bound():
    """the height field's slot of a row: its world position, the model's axes, the half-extents and elevation scale, the compiler's bound"""
    e = TerrainSim(terrain_bank(1, 1))
    pos, size = placement(2)
    row, base = e.row(pos, size).reshape(16, 16), e.row().reshape(16, 16)
    import camera_support as CS
    sc = hf_scene(CS.EmuCam('cassie_hfield').scene(), pos, size)
    k = sc.slot('hfield1')
    assert np.allclose(row[k, :3], sc.pos[k], atol=1e-15) and np.array_equal(row[k, 3:12], base[k, 3:12])
    assert np.array_equal(row[k, 12:15], size[:3]) and row[k, 15] == rbound(size)
    assert np.array_equal(np.delete(row, k, axis=0), np.delete(base, k, axis=0))
    assert e.set(2, 0, size=[1, 0, 0.1, 0.1]) == -1 and e.set(2, 0, size=[1, 1, -0.1, 0.1]) == -1 and e.set(2, 0, size=[1, 1, 0.1, np.nan]) == -1


# ------------------------------------------------------------------ 3. rays and depth images against their oracles
def _placements(n, rng):
    t = rng.integers(0, 4, n).astype(np.int32)
    pos = np.array([placement(i)[0] for i in range(n)])
    size = np.array([placement(i)[1] * [1, 1, rng.uniform(0, 2), 1] for i in range(n)])
    return t, pos, size


@pytest.mark.parametrize('fp32', [False, True])
def test_rays_follow_the_oracle(fp32):
    """a height scan and slanted rays in the world frame over 8 environments with their own terrain, scale and position: fp64 within 1e-12 of the ray
    oracle given the same terrain and placement; fp32 equal slots and within 1e-5 * max outside the rays whose outcome flips under a 1e-5 m nudge"""
    rng = np.random.default_rng(4)
    bank = terrain_bank(4, 23)
    n = 8
    t, pos, size = _placements(n, rng)
    e = TerrainSim(bank, fp32)
    genv = np.array([e.row(pos[i], size[i]) for i in range(n)])
    org, dirs = RS.height_scan(np.linspace(-1.5, 1.5, 9), np.linspace(-1.2, 1.2, 7), z_start=1.0)
    slant = rng.normal(size=(24, 3)) * [1, 1, 0.2] + [0, 0, -1]
    org = np.concatenate([org, rng.uniform(-2, 2, (24, 3)) * [1, 1, 0] + [0, 0, 1.0]])
    dirs = np.concatenate([dirs, slant / np.linalg.norm(slant, axis=1)[:, None]])
    k, maxd = len(org), 4.0
    out = np.zeros((n, k, 4))
    q = np.zeros((n, 35))
    q[:, 3] = 1
    frame = np.full(k, RS.WORLD, dtype=np.int32)
    assert e.L.emu_tr_ray_cast(e.h, n, _dp(q), 35, _dp(genv), t.ctypes.data_as(C.POINTER(C.c_int)), frame.ctypes.data_as(C.POINTER(C.c_int)), _dp(org), _dp(dirs),
                               _dp(np.full(k, maxd)), k, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
    import camera_support as CS
    sc0 = CS.EmuCam('cassie_hfield').scene()   # every static slot, in slot order
    hits = 0
    for i in range(n):
        sc = hf_scene(sc0, pos[i], size[i])
        ref = RS.oracle_cast(sc, org, dirs, maxd, bank[t[i]].astype(np.float64))
        hits += (ref[:, 0] >= 0).sum()
        if not fp32:
            assert np.abs(out[i] - ref).max() <= 1e-12, (i, np.abs(out[i] - ref).max())
            continue
        amb = RS.ambiguous(sc, org, dirs, maxd, bank[t[i]].astype(np.float64))
        assert amb.mean() < 0.05
        assert np.array_equal(out[i][~amb, 2], ref[~amb, 2]) and np.abs(out[i][~amb] - ref[~amb]).max() <= 1e-5 * maxd
    assert hits > 0.8 * n * k
    e.close()


@pytest.mark.parametrize('fp32', [False, True])
def test_depth_images_follow_the_oracle(fp32):
    """the egocentric camera of cassie_hfield at standing, mid-fall and crossed-leg states, each environment on its own terrain, scale and position:
    fp64 within 1e-12 of the camera oracle; fp32 within 1e-5 * zfar outside the pixels whose outcome flips under a 1e-5 m nudge"""
    import camera_support as CS
    import test_camera as TC
    rng = np.random.default_rng(12)
    bank = terrain_bank(4, 29)
    cam = CS.EmuCam('cassie_hfield', fp32)
    body, cpos_b, cquat, fovy, zfar = TC.camera_of('cassie_hfield', cam)
    qs = TC.states('cassie_hfield', rng)
    n = len(qs)
    t, pos, size = _placements(n, rng)
    e = TerrainSim(bank, fp32)
    genv = np.array([e.row(pos[i], size[i]) for i in range(n)])
    W, H = 24, 18
    out = np.zeros((n, H, W))
    q = np.array(qs)
    assert e.L.emu_tr_render(e.h, n, _dp(q), q.shape[1], _dp(genv), t.ctypes.data_as(C.POINTER(C.c_int)), body, _dp(cpos_b), _dp(cquat), fovy, W, H, zfar,
                             out.ctypes.data_as(C.POINTER(C.c_double))) == 0
    sc0 = cam.scene()
    for i in range(n):
        xpos, xquat = CS.oracle_poses('cassie_hfield', qs[i])
        mv = CS.Moving(cam.table, cam.moving_geoms, xpos, xquat)
        cp, cR = CS.camera_world(xpos, xquat, body, cpos_b, cquat / np.linalg.norm(cquat))
        sc = hf_scene(sc0, pos[i], size[i])
        hf = bank[t[i]].astype(np.float64)
        a, ga = CS.oracle_render(sc, mv, cp, cR, fovy, W, H, zfar, hf)
        assert (ga >= 0).mean() > 0.3
        if not fp32:
            assert np.abs(out[i] - a).max() <= 1e-12, np.abs(out[i] - a).max()
            continue
        amb = CS.ambiguous(sc, mv, cp, cR, fovy, W, H, zfar, hf)
        assert amb.mean() < 0.005, amb.mean()
        assert np.abs(out[i] - a)[~amb].max() <= 1e-5 * zfar
    cam.close()
    e.close()
