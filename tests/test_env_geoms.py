"""Per-environment placement of the static planes / boxes (cassie_batch_set_env_geom_pose): the product's stepper source in the host emulation, with the
placement held in the environment's geom row (the F_EG instance) instead of the model block.  The GPU twins are in tests/test_gpu_env_geoms.py.

The emulation with a geom row is tests/emu/emu_env_geoms.cpp (emu.cpp plus the row), built into its own library here.  The oracle's bounding radius
of a resized box (the per-environment rule |size|) is given to it through a temporary copy of its model table."""
import ctypes as C
import os
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from test_model_variants import PD_ROW, STAIRS

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
TILT = np.deg2rad(5.0)
FLOOR_TILT = ('floor', None, [np.cos(TILT / 2), np.sin(TILT / 2), 0, 0], None)    # the floor turned 5 degrees about x: one foot higher than the other
# a box far longer than its file size (half-sizes 1 1 1): its centre is 2.9 m ahead, its near end under the left foot.  With the file's bounding radius
# (sqrt 3) it would be culled by the broad phase; the per-environment radius |size| keeps it
LONG_BOX = ('box1', [2.9, 0.135, -0.02], None, [3.0, 0.1, 0.05])
GEOM_ID = {'floor': 0, **{'box%d' % i: i for i in range(1, 16)}}   # cassie.xml's static geoms, in the reference's numbering

_EG_LIB = None


def eg_lib():
    """the emulation library with the per-environment geom row (tests/emu/emu_env_geoms.cpp + the MJCF loader)"""
    global _EG_LIB
    if _EG_LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_env_geoms.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_env_geoms.cpp'), os.path.join(E.CSRC, 'mjcf.cpp'), os.path.join(E.HERE, 'emu', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], srcs[1]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_eg_new.restype = vp
        L.emu_eg_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_eg_free', 'emu_eg_enable', 'emu_eg_forward', 'emu_plain'):
            getattr(L, n).argtypes = [vp]
        L.emu_eg_set.argtypes = [vp, ci, dp, dp, dp]
        L.emu_eg_step.argtypes = [vp, dp, ci]
        L.emu_eg_row.argtypes = L.emu_eg_block_wpose.argtypes = [vp, dp]
        L.emu_eg_geom_slot.argtypes = [vp, ci]
        L.emu_eg_static_wpose.argtypes = [vp, ci, dp]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set_geom.argtypes = [vp, ci, dp, dp, dp]
        L.emu_geom_id.argtypes = [vp, C.c_char_p]
        _EG_LIB = L
    return _EG_LIB


def _dp(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


class GeomRowSim:
    """one emulated environment; set_env_geom places a static plane / box through its geom row only, from then on the F_EG path runs"""

    def __init__(self, model_path, fp32=False):
        self.L = eg_lib()
        self.h = self.L.emu_eg_new(model_path.encode(), 1 if fp32 else 0)
        assert self.h, model_path

    def close(self):
        if self.h:
            self.L.emu_eg_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def plain(self):
        self.L.emu_plain(self.h)

    def step(self, pd50, nticks=1):
        self.L.emu_eg_step(self.h, _dp(pd50), nticks)

    def forward(self):
        self.L.emu_eg_forward(self.h)

    def set_geom(self, name, pos=None, quat=None, size=None):
        """the shared placement: move the geom in the model block (cassie_sim_set_geom_name_*)"""
        g = self.L.emu_geom_id(self.h, name.encode())
        assert self.L.emu_set_geom(self.h, g, _dp(pos), _dp(quat), _dp(size)) == 0, name
        return g

    def set_env_geom(self, name, pos=None, quat=None, size=None):
        g = self.L.emu_geom_id(self.h, name.encode())
        assert self.L.emu_eg_set(self.h, g, _dp(pos), _dp(quat), _dp(size)) == 0, name
        return g

    def enable_env_geoms(self):
        self.L.emu_eg_enable(self.h)

    def row(self):
        out = np.zeros(256)
        self.L.emu_eg_row(self.h, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def block_wpose(self):
        out = np.zeros(16 * 12)
        self.L.emu_eg_block_wpose(self.h, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def geom_slot(self, g):
        return self.L.emu_eg_geom_slot(self.h, g)

    def static_wpose(self, g):
        out = np.zeros(12)
        self.L.emu_eg_static_wpose(self.h, g, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out


def placed_oracle(O, placements):
    """an oracle of cassie.xml with `placements` [(name, pos, quat, size)]; a resized geom's bounding radius is |size|, as the per-environment verb
    sets it (written into a temporary copy of the model table: the oracle reads geom_rbound from there)"""
    path = os.path.join(GOLDEN, 'cassie.omodel')
    rb = {GEOM_ID[name]: float(np.linalg.norm(size)) for name, _, _, size in placements if size is not None}
    if rb:
        lines = open(path).read().split('\n')
        for i, ln in enumerate(lines):
            if ln.startswith('geom_rbound '):
                t = ln.split()
                for g, r in rb.items():
                    t[3 + g] = repr(r)
                lines[i] = ' '.join(t)
        with tempfile.TemporaryDirectory() as d:
            p = os.path.join(d, 'cassie.omodel')
            with open(p, 'w') as f:
                f.write('\n'.join(lines))
            o = O.OracleSim(p)
    else:
        o = O.OracleSim(path)
    for name, pos, quat, size in placements:
        g = GEOM_ID[name]
        if pos is not None:
            o.model_arr('geom_pos').reshape(-1, 3)[g] = pos
        if quat is not None:
            o.model_arr('geom_quat').reshape(-1, 4)[g] = quat
        if size is not None:
            o.model_arr('geom_size').reshape(-1, 3)[g] = size
    o.forward()
    return o


def _run_pair(oracle_mod, placements, fp32, nticks=700):
    """an oracle and an emulated environment with `placements` [(name, pos, quat, size)] given to the environment's geom row only"""
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    e = GeomRowSim(os.path.join(MODELS, 'cassie.cmodel'), fp32=fp32)
    e.plain()
    for name, pos, quat, size in placements:
        e.set_env_geom(name, pos=pos, quat=quat, size=size)
    o = placed_oracle(oracle_mod, placements)
    e.forward()
    worst, iters_equal, contacts = 0.0, True, set()
    for k in range(nticks):
        o.step_pd(u)
        e.step(PD_ROW)
        worst = max(worst, np.abs(e.get('qpos')[:35] - o.arr('qpos')).max())
        iters_equal = iters_equal and int(e.get('counters')[3]) == o.get_int('solver_iter')
        contacts.update(g for c in o.contacts() for g in (c['geom1'], c['geom2']) if g < 16)   # static geoms met: floor 0, boxes 1..15
    assert int(e.get('counters')[4]) == 0   # no dropped contacts
    return o, e, worst, iters_equal, contacts


@pytest.mark.parametrize('fp32', [False, True])
def test_row_placement_is_bitwise_the_shared_placement(fp32):
    """the stairs of test_model_variants placed through the geom row only run the F_EG path; the result is bitwise the shared-placement path's"""
    a, b = GeomRowSim(os.path.join(MODELS, 'cassie.cmodel'), fp32=fp32), GeomRowSim(os.path.join(MODELS, 'cassie.cmodel'), fp32=fp32)
    a.plain()
    b.plain()
    for name, pos, quat, size in STAIRS:
        a.set_geom(name, pos=pos, quat=quat, size=size)
        b.set_env_geom(name, pos=pos, quat=quat, size=size)
    a.forward()
    b.forward()
    for k in range(700):
        a.step(PD_ROW)
        b.step(PD_ROW)
        for f in ('qpos', 'qvel', 'obs', 'counters'):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    assert int(b.get('counters')[4]) == 0


@pytest.mark.parametrize('case', ['tilted_floor', 'long_box', 'box_and_floor'])
def test_row_only_placement_follows_the_oracle(oracle_mod, case):
    placements = {'tilted_floor': [FLOOR_TILT], 'long_box': [LONG_BOX], 'box_and_floor': [STAIRS[0]]}[case]
    for fp32, tol in ((False, 1e-10), (True, 1e-4)):
        o, e, worst, iters_equal, contacts = _run_pair(oracle_mod, placements, fp32)
        assert worst < tol, (case, fp32, worst)
        assert iters_equal or fp32, case   # fp64: the same PGS iteration count as the oracle every tick
        if case == 'tilted_floor':
            assert contacts == {0}
        else:
            assert 1 in contacts and (case == 'long_box' or 0 in contacts), contacts   # box contacts (left foot); box_and_floor: the right foot on the floor


def test_box_and_floor_contacts_interleave_in_mujoco_order(oracle_mod):
    """one foot on a row-placed box, the other on the floor: the left foot's box contact comes before the right foot's floor contact in MuJoCo's order
    although the kernel visits the static-box pairs in a second run"""
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    e = GeomRowSim(os.path.join(MODELS, 'cassie.cmodel'))
    name, pos, _, size = STAIRS[0]
    e.set_env_geom(name, pos=pos, size=size)
    o = placed_oracle(oracle_mod, [(name, pos, None, size)])
    e.forward()
    mixed = False
    for k in range(500):
        o.step_pd(u)
        e.step(PD_ROW)
        gs = [c['geom1'] for c in o.contacts()]
        mixed = mixed or (0 in gs and any(x != 0 for x in gs) and gs != sorted(gs))
        assert int(e.get('counters')[3]) == o.get_int('solver_iter'), k
    assert np.abs(e.get('qpos')[:35] - o.arr('qpos')).max() < 1e-10 and mixed


@pytest.mark.parametrize('model', sorted(f[:-7] for f in os.listdir(MODELS) if f.endswith('.cmodel')))
def test_pose_helper_reproduces_the_model_block(model):
    """the world-pose composition shared by the model block builder and the per-environment verbs gives the block's geom_wpose exactly, for every
    static collision geom, in both precisions"""
    for fp32 in (False, True):
        e = GeomRowSim(os.path.join(MODELS, model + '.cmodel'), fp32=fp32)
        block = e.block_wpose().reshape(16, 12)
        n = 0
        for g in range(256):
            k = e.geom_slot(g)
            if k < 16:
                continue
            w = e.static_wpose(g)
            assert np.array_equal(w.astype(np.float32).astype(np.float64) if fp32 else w, block[k - 16]), (model, g)
            n += 1
        assert n >= 1
        e.close()


def test_fresh_row_holds_the_model_placement():
    """the row a batch starts from is the block's own placement: slot k = world pose, size, bounding radius of device geom 16 + k"""
    e = GeomRowSim(os.path.join(MODELS, 'cassie.cmodel'))
    e.enable_env_geoms()
    row, block = e.row().reshape(16, 16), e.block_wpose().reshape(16, 12)
    assert np.array_equal(row[:, :12], block)
    g = e.set_env_geom(LONG_BOX[0], size=LONG_BOX[3])
    assert e.row().reshape(16, 16)[e.geom_slot(g) - 16, 15] == np.linalg.norm(LONG_BOX[3])
    e.close()


def test_oracle_model_copy_carries_the_bound(oracle_mod):
    """the long box needs its |size| bound in the oracle too: with the file's bound the oracle culls the foot / box pairs and the foot sinks through"""
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    stale = oracle_mod.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    stale.model_arr('geom_pos').reshape(-1, 3)[1] = LONG_BOX[1]
    stale.model_arr('geom_size').reshape(-1, 3)[1] = LONG_BOX[3]
    stale.forward()
    placed = placed_oracle(oracle_mod, [LONG_BOX])
    met = [set(), set()]
    for k in range(300):
        for i, o in enumerate((stale, placed)):
            o.step_pd(u)
            met[i].update(g for c in o.contacts() for g in (c['geom1'], c['geom2']) if g < 16)
    assert 1 not in met[0] and 1 in met[1], met
