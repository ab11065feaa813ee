"""Per-environment body offsets (cassie_batch_set_env_body_pos): the product's stepper, ray and camera sources in the host emulation, with each body's
position in its parent frame taken from the environment's row (the F_BP instances) instead of the model block.  The GPU twins are in
tests/test_gpu_env_body_pos.py.

The emulation is tests/emu/emu_env_body_pos.cpp, built into its own library here.  The fp64 oracle gets the offsets through a temporary copy of its
model table (MuJoCo's body_pos; nothing else in the table changes, as when the reference writes m->body_pos)."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
CE_BINVW, CE_DINVW, CE_PGS = 192, 224, 258   # devmodel.h CE_*

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_env_body_pos.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_env_body_pos.cpp', 'emu_camera.cpp', 'emu_raycast.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'raycast.inl', 'camera.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci, ip = C.c_void_p, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int)
        L.emu_bp_new.restype = vp
        L.emu_bp_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_bp_free', 'emu_bp_forward', 'emu_bp_set_const', 'emu_plain'):
            getattr(L, n).argtypes = [vp]
        L.emu_bp_set.argtypes = L.emu_bp_set_model.argtypes = [vp, dp]
        L.emu_bp_step.argtypes = [vp, dp, ci]
        L.emu_bp_rays.argtypes = [vp, ip, dp, dp, dp, ci, dp]
        L.emu_bp_camera.argtypes = [vp, ci, dp, dp, C.c_double, ci, ci, C.c_double, dp]
        L.emu_bp_reach.argtypes = [vp, dp, dp]
        L.emu_bp_refused.argtypes = [vp, ci]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


class BodyRowSim:
    """one emulated environment; set_env_body_pos fills its row, from then on the F_BP source runs"""

    def __init__(self, model, fp32=False):
        self.L = lib()
        self.h = self.L.emu_bp_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h

    def close(self):
        if self.h:
            self.L.emu_bp_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def set_env_body_pos(self, pos):
        self._keep = np.ascontiguousarray(pos, dtype=np.float64)
        self.L.emu_bp_set(self.h, _dp(self._keep))

    def step(self, pd50, nticks=1):
        self.L.emu_bp_step(self.h, _dp(pd50), nticks)

    def forward(self):
        self.L.emu_bp_forward(self.h)

    def set_const(self):
        self.L.emu_bp_set_const(self.h)


def table(model):
    """(names_body, nbody, body_pos [nbody, 3], body_weldid) of the oracle's model table"""
    t = {ln.split()[0]: ln.split()[3:] for ln in open(os.path.join(GOLDEN, model + '.omodel')).read().split('\n') if ln.strip()}
    names = t['names_body']
    return names, len(names), np.array([float(x) for x in t['body_pos']]).reshape(-1, 3), np.array([int(x) for x in t['body_weldid']])


def oracle_with(O, model, body_pos, rbound=None):
    """an fp64 oracle of `model` whose body_pos is `body_pos` [nbody, 3]; rbound {geom: bounding radius} overrides geom_rbound (a box placed per
    environment gets |size|, as cassie_batch_set_env_geom_pose sets it)"""
    path = os.path.join(GOLDEN, model + '.omodel')
    lines = open(path).read().split('\n')
    for i, ln in enumerate(lines):
        t = ln.split()
        if ln.startswith('body_pos '):
            lines[i] = ' '.join(t[:3] + [repr(float(x)) for x in np.asarray(body_pos, float).ravel()])
        elif ln.startswith('geom_rbound ') and rbound:
            for g, r in rbound.items():
                t[3 + g] = repr(float(r))
            lines[i] = ' '.join(t)
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, model + '.omodel')
        with open(p, 'w') as f:
            f.write('\n'.join(lines))
        return O.OracleSim(p)


def offsets(model, seed):
    """seeded offsets of the kinds users randomise: cassie -- hip roll / hip pitch +-5 mm and one loop body (the left tarsus) +-2 mm; cassie_mass -- the
    welded load +-2 cm; cassie_tray_box -- the tray +-1 cm"""
    names, nb, bp, _ = table(model)
    rng = np.random.default_rng(seed)
    p = bp.copy()
    if model == 'cassie':
        for n in ('left-hip-roll', 'right-hip-roll', 'left-hip-pitch', 'right-hip-pitch'):
            p[names.index(n)] += rng.uniform(-0.005, 0.005, 3)
        p[names.index('left-tarsus')] += rng.uniform(-0.002, 0.002, 3)
    elif model == 'cassie_mass':
        p[names.index('load_mass')] += rng.uniform(-0.02, 0.02, 3)
    else:
        p[names.index('tray')] += rng.uniform(-0.01, 0.01, 3)
    return p


# ------------------------------------------------------------------ 1. rows at the model's values are the counterpart source, bitwise
@pytest.mark.parametrize('fp32', [False, True])
def test_model_rows_are_bitwise_the_counterpart(fp32):
    _, _, bp, _ = table('cassie')
    a, b = BodyRowSim('cassie', fp32), BodyRowSim('cassie', fp32)
    b.set_env_body_pos(bp)
    b.forward()
    for k in range(400):
        a.step(PD_ROW)
        b.step(PD_ROW)
        for f in ('qpos', 'qvel', 'obs', 'aux', 'counters'):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    a.close()
    b.close()


# ------------------------------------------------------------------ 2. against the oracle
@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box'])
def test_env_body_pos_follows_the_oracle(oracle_mod, model):
    """fp64: qpos within 1e-9 of the oracle with the same body_pos over 500 ticks, the same PGS iteration count every tick"""
    p = offsets(model, 5)
    o = oracle_with(oracle_mod, model, p)
    e = BodyRowSim(model)
    e.set_env_body_pos(p)
    e.forward()
    o.forward()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    worst, iters_equal = 0.0, True
    for k in range(500):
        o.step_pd(u)
        e.step(PD_ROW)
        worst = max(worst, np.abs(e.get('qpos')[:o.nq] - o.arr('qpos')).max())
        iters_equal = iters_equal and int(e.get('counters')[3]) == o.get_int('solver_iter')
    assert worst < 1e-9 and iters_equal, (model, worst, iters_equal)
    # the offsets change the motion: the model's own trajectory is elsewhere
    o0 = oracle_mod.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    for k in range(500):
        o0.step_pd(u)
    assert np.abs(o0.arr('qpos') - o.arr('qpos')).max() > 1e-5
    e.close()
    o.close()
    o0.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_mass'])
def test_set_const_rows_follow_the_oracle(oracle_mod, model):
    """mode 3 at qpos0 with the environment's offsets: the invweights and the PGS scale match the oracle's mj_setConst with the same body_pos"""
    p = offsets(model, 9)
    o = oracle_with(oracle_mod, model, p)
    e = BodyRowSim(model)
    e.set_env_body_pos(p)
    e.set_const()
    o.just_set_const()
    nb, nv = o.get_int('nbody'), o.get_int('nv')
    c = e.get('cenv')
    assert np.abs(c[CE_BINVW:CE_BINVW + nb] - o.model_arr('body_invweight0')[0::2]).max() < 1e-12
    assert np.abs(c[CE_DINVW:CE_DINVW + 32] / o.model_arr('dof_invweight0')[:32] - 1).max() < 1e-12
    assert abs(c[CE_PGS] * o.model_arr('meaninertia')[0] * nv - 1) < 1e-12
    # and they differ from the model's constants: the offsets moved the loads
    ref = oracle_mod.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    ref.just_set_const()
    assert np.abs(ref.model_arr('dof_invweight0') - o.model_arr('dof_invweight0')).max() > 1e-9
    e.close()
    o.close()
    ref.close()


# ------------------------------------------------------------------ 3. the row is the model block with those offsets (rays, cameras, broad phase)
@pytest.mark.parametrize('fp32', [False, True])
def test_rays_and_camera_read_the_row(fp32):
    """a per-environment pelvis offset through the row gives bitwise the height scan and depth image of the same offset in the model block (the ray and
    camera sources' model-block path is the one held to the ray and camera oracles); without a row the outputs are the model's"""
    names, nb, bp, _ = table('cassie')
    p = bp.copy()
    p[names.index('cassie-pelvis')] += [0.03, -0.02, 0.05]
    k = 24
    ang = np.linspace(0, 2 * np.pi, k, endpoint=False)
    frame = np.ones(k, dtype=np.int32)   # RAY_ROOT: rays fixed to the root body move with its offset
    org = np.stack([0.3 * np.cos(ang), 0.3 * np.sin(ang), np.zeros(k)], 1)
    dirs = np.tile([0.0, 0.0, -1.0], (k, 1))
    maxd = np.full(k, 3.0)

    def scan(s):
        out = np.zeros(k * 4)
        assert s.L.emu_bp_rays(s.h, frame.ctypes.data_as(C.POINTER(C.c_int)), _dp(org), _dp(dirs), _dp(maxd), k, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
        return out

    def depth(s):
        out = np.zeros(24 * 16)
        assert s.L.emu_bp_camera(s.h, names.index('cassie-pelvis'), _dp([0.1, 0, 0.1]), _dp([0.5, -0.5, 0.5, -0.5]), 70.0, 24, 16, 5.0, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
        return out

    row, block, none = (BodyRowSim('cassie', fp32) for _ in range(3))
    row.set_env_body_pos(p)
    assert block.L.emu_bp_set_model(block.h, _dp(p)) == 0
    for s in (row, block, none):
        s.forward()
    assert np.array_equal(scan(row), scan(block)) and np.array_equal(depth(row), depth(block))
    assert not np.array_equal(scan(row), scan(none))
    assert np.abs(depth(row) - depth(none)).max() > 1e-3
    for s in (row, block, none):
        s.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box'])
def test_robot_reach_rule(model):
    """robot_reach_of with the model's offsets is build_dev_model's bound bitwise (the batch's setter takes the largest over its rows); a longer
    tarsus lengthens it"""
    names, nb, bp, _ = table(model)
    for fp32 in (0, 1):
        s = BodyRowSim(model, bool(fp32))
        out = np.zeros(2)
        s.L.emu_bp_reach(s.h, _dp(bp), out.ctypes.data_as(C.POINTER(C.c_double)))
        assert out[0] == out[1], (model, fp32, out)
        p = bp.copy()
        p[names.index('left-tarsus')] *= 1.3
        s.L.emu_bp_reach(s.h, _dp(p), out.ctypes.data_as(C.POINTER(C.c_double)))
        assert out[1] > out[0] + 0.05, out
        s.close()


@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_refused_bodies(model):
    """the verb refuses the world body, bodies welded to the world and the extra free body, and nothing else"""
    names, nb, _, weld = table(model)
    s = BodyRowSim(model)
    xb = nb - 1 if model == 'cassie_tray_box' else -1
    got = [s.L.emu_bp_refused(s.h, b) for b in range(nb)]
    assert got == [1 if (b == 0 or weld[b] == 0 or b == xb) else 0 for b in range(nb)]
    s.close()
