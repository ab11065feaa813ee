"""Shared pieces of the ray-casting tests: the TEST-ONLY fp64 ray oracle (tests/ray_oracle.c) and host emulation of the ray source
(tests/emu/emu_raycast.cpp), each built into its own library, and the scenes both are given.

The oracle takes world rays and the static geoms in world coordinates.  The root pose that places heading- and root-frame rays comes from the fp64
oracle stepper's own kinematics (xpos / xquat of the root body), the static geoms from the model table or from the placement a test chooses."""
import ctypes as C
import os
import subprocess

import numpy as np

from emu_harness import CSRC, HERE, REPO

BUILD = os.path.join(HERE, 'emu', '_build')
GOLDEN = os.path.join(HERE, 'golden')
MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
HEADING, ROOT, WORLD = 0, 1, 2
dp = C.POINTER(C.c_double)


def _build(out, srcs, cmd):
    if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(s) for s in srcs):
        os.makedirs(BUILD, exist_ok=True)
        subprocess.check_call(cmd + ['-o', out + '.tmp'])
        os.replace(out + '.tmp', out)
    return C.CDLL(out)


_libs = {}


def oracle_lib():
    if 'o' not in _libs:
        src = os.path.join(HERE, 'ray_oracle.c')
        L = _build(os.path.join(BUILD, 'libray_oracle.so'), [src], ['gcc', '-O1', '-std=c99', '-fPIC', '-shared', src, '-lm'])
        L.oracle_raycast.argtypes = [C.c_int, C.POINTER(C.c_int), dp, dp, dp, dp, C.c_int, C.c_int, dp, C.c_int, dp, dp, dp, dp]
        _libs['o'] = L
    return _libs['o']


def emu_lib():
    if 'e' not in _libs:
        src = os.path.join(HERE, 'emu', 'emu_raycast.cpp')
        deps = [src, os.path.join(HERE, 'emu', 'emu.cpp'), os.path.join(CSRC, 'raycast.inl'), os.path.join(CSRC, 'step_core.inl'), os.path.join(CSRC, 'devbuild.h'),
                os.path.join(CSRC, 'devmodel.h'), os.path.join(CSRC, 'mjcf.cpp'), os.path.join(CSRC, 'model.h')]
        L = _build(os.path.join(BUILD, 'libcassie_emu_raycast.so'), deps, ['g++', '-O1', '-std=c++17', '-fPIC', '-shared', src, os.path.join(CSRC, 'mjcf.cpp')])
        L.emu_new.restype = C.c_void_p
        L.emu_new.argtypes = [C.c_char_p, C.c_int]
        L.emu_free.argtypes = [C.c_void_p]
        L.emu_forward.argtypes = [C.c_void_p]
        L.emu_set.argtypes = [C.c_void_p, C.c_char_p, dp, C.c_int]
        L.emu_get.argtypes = [C.c_void_p, C.c_char_p, dp, C.c_int]
        L.emu_set_hfield.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_int]
        L.emu_ray_cast.argtypes = [C.c_void_p, C.c_int, dp, C.c_int, dp, C.POINTER(C.c_float), C.c_int, C.POINTER(C.c_int), dp, dp, dp, C.c_int, dp]
        L.emu_ray_root.argtypes = [C.c_void_p, dp]
        L.emu_ray_slots.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
        L.emu_ray_genv0.argtypes = [C.c_void_p, dp]
        _libs['e'] = L
    return _libs['e']


def _d(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def load_table(path):
    d = {}
    for line in open(path):
        if line[0] == '#':
            continue
        t = line.split()
        d[t[0]] = t[3:3 + int(t[2])] if t[1] == 'S' else np.array([float(x) for x in t[3:3 + int(t[2])]])
    return d


def quat2mat(q):
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[w*w+x*x-y*y-z*z, 2*(x*y-w*z), 2*(x*z+w*y)], [2*(x*y+w*z), w*w-x*x+y*y-z*z, 2*(y*z-w*x)], [2*(x*z-w*y), 2*(y*z+w*x), w*w-x*x-y*y+z*z]])


class Scene:
    """the static geoms of a model in collision-slot order (world pose, size, type) and its height field; place() moves a plane / box as
    cassie_batch_set_env_geom_pose does for a geom of the world body."""

    def __init__(self, name, slots):
        self.t = load_table(os.path.join(MODELS, name + '.cmodel'))
        t = self.t
        self.slots = [g for g in slots if g >= 0]
        self.type = np.array([int(t['geom_type'][g]) for g in self.slots], dtype=np.int32)
        self.pos, self.R = [], []
        for g in self.slots:   # on the world body, or on a body welded to it (the height field's floor body)
            b = int(t['geom_bodyid'][g])
            Rb, pb = (np.eye(3), np.zeros(3)) if b == 0 else (quat2mat(t['body_quat'][4 * b:4 * b + 4]), t['body_pos'][3 * b:3 * b + 3])
            assert b == 0 or (int(t['body_parentid'][b]) == 0 and int(t['body_jntnum'][b]) == 0)
            self.pos.append(pb + Rb @ t['geom_pos'][3 * g:3 * g + 3])
            self.R.append(Rb @ quat2mat(t['geom_quat'][4 * g:4 * g + 4]))
        self.pos, self.R = np.array(self.pos), np.array(self.R)
        self.size = np.array([t['geom_size'][3 * g:3 * g + 3] for g in self.slots])
        self.nrow = int(t['hfield_nrow'][0]) if t['hfield_nrow'].size else 0
        self.ncol = int(t['hfield_ncol'][0]) if t['hfield_ncol'].size else 0
        self.hsize = _d(t['hfield_size'][:4]) if t['hfield_size'].size else np.zeros(4)
        self.hf = None

    def copy(self):
        s = Scene.__new__(Scene)
        s.__dict__.update(self.__dict__)
        s.pos, s.R, s.size = self.pos.copy(), self.R.copy(), self.size.copy()
        return s

    def slot(self, name):
        return self.slots.index(self.t['names_geom'].index(name))

    def place(self, name, pos=None, quat=None, size=None):
        k = self.slot(name)
        if pos is not None:
            self.pos[k] = pos
        if quat is not None:
            self.R[k] = quat2mat(quat)
        if size is not None:
            self.size[k] = size
        return k

    def genv_row(self):
        """this placement as a GEOM_ENV_W row (position, z, x, y axes, size, bounding radius per slot)"""
        row = np.zeros(256)
        for k in range(len(self.slots)):
            R = self.R[k]
            row[16 * k:16 * k + 12] = np.concatenate([self.pos[k], R[:, 2], R[:, 0], R[:, 1]])
            row[16 * k + 12:16 * k + 15] = self.size[k]
            row[16 * k + 15] = np.linalg.norm(self.size[k]) if self.type[k] == 6 else 0.0
        return row


def world_rays(kind, org, dirs, root_pos, root_R):
    """rays of one frame kind in world coordinates (the heading frame: the root's position and the yaw of its x axis)"""
    org, dirs = np.atleast_2d(_d(org)), np.atleast_2d(_d(dirs))
    dirs = dirs / np.linalg.norm(dirs, axis=1)[:, None]
    if kind == WORLD:
        return org, dirs
    if kind == ROOT:
        M = root_R
    else:
        c, s = root_R[0, 0], root_R[1, 0]
        h = np.hypot(c, s)
        c, s = (c / h, s / h) if h > 1e-15 else (1.0, 0.0)
        M = np.array([[c, -s, 0], [s, c, 0], [0, 0, 1.0]])
    return root_pos + org @ M.T, dirs @ M.T


def oracle_cast(scene, org_w, dir_w, maxd, hf=None):
    """[k][4] rows of the fp64 oracle for world rays"""
    L = oracle_lib()
    k = len(org_w)
    out = np.zeros((k, 4))
    pos, R, size = _d(scene.pos), _d(scene.R), _d(scene.size)
    h = None if hf is None else _d(hf)
    L.oracle_raycast(len(scene.slots), scene.type.ctypes.data_as(C.POINTER(C.c_int)), pos.ctypes.data_as(dp), R.ctypes.data_as(dp), size.ctypes.data_as(dp),
                     None if h is None else h.ctypes.data_as(dp), scene.nrow, scene.ncol, scene.hsize.ctypes.data_as(dp), k,
                     _d(org_w).ctypes.data_as(dp), _d(dir_w).ctypes.data_as(dp), _d(np.broadcast_to(maxd, (k,))).ctypes.data_as(dp), out.ctypes.data_as(dp))
    return out


def root_pose(osim, body):
    """the root body's (the pelvis) world position and rotation from the oracle's forward kinematics"""
    return np.array(osim.arr('xpos')[3 * body:3 * body + 3]), quat2mat(osim.arr('xquat')[4 * body:4 * body + 4])


def height_scan(xs, ys, z_start=1.0):
    """the scan pattern of CassieBatch.set_height_scan: origins on the grid z_start above the root, rays along -z"""
    gx, gy = np.meshgrid(np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64), indexing='ij')
    org = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, float(z_start))], axis=1)
    return org, np.tile([0.0, 0.0, -1.0], (len(org), 1))


def ambiguous(scene, org_w, dir_w, maxd, hf=None, nudge=1e-5):
    """rays whose hit / miss or geom changes in the oracle when the origin moves by +-nudge in x or y (edge grazes)"""
    base = oracle_cast(scene, org_w, dir_w, maxd, hf)
    amb = np.zeros(len(org_w), dtype=bool)
    for ax in (0, 1):
        for s in (-nudge, nudge):
            o = _d(org_w).copy()
            o[:, ax] += s
            r = oracle_cast(scene, o, dir_w, maxd, hf)
            amb |= ((r[:, 0] >= 0) != (base[:, 0] >= 0)) | (r[:, 2] != base[:, 2])
    return amb
