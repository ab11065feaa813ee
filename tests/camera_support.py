"""Shared pieces of the depth-camera tests: the TEST-ONLY fp64 camera oracle (tests/camera_oracle.c) and host emulation of the camera source
(tests/emu/emu_camera.cpp), each built into its own library, and the scenes both are given.

The oracle takes the camera and every geom in world coordinates.  Body poses come from the fp64 oracle stepper's own kinematics (xpos / xquat), the
static geoms from the model table or from the placement a test chooses (raycast_support.Scene), the moving geoms from the model table's geom frames on
those body poses, the camera from the table's <camera> entries or from the mount a test chooses."""
import ctypes as C
import os

import numpy as np

import oracle as O
import raycast_support as RS
from raycast_support import BUILD, GOLDEN, MODELS, _build, _d, dp, quat2mat
from emu_harness import CSRC, HERE

ip = C.POINTER(C.c_int)
_libs = {}


def oracle_lib():
    if 'o' not in _libs:
        srcs = [os.path.join(HERE, 'camera_oracle.c'), os.path.join(HERE, 'ray_oracle.c')]
        L = _build(os.path.join(BUILD, 'libcamera_oracle.so'), srcs, ['gcc', '-O1', '-std=c99', '-fPIC', '-shared', srcs[0], '-lm'])
        L.oracle_camera.argtypes = [C.c_int, ip, dp, dp, dp, dp, C.c_int, C.c_int, dp, C.c_int, ip, dp, dp, dp, dp, dp, C.c_double, C.c_int, C.c_int,
                                    C.c_double, dp, ip]
        _libs['o'] = L
    return _libs['o']


def emu_lib():
    if 'e' not in _libs:
        src = os.path.join(HERE, 'emu', 'emu_camera.cpp')
        deps = [src, os.path.join(HERE, 'emu', 'emu.cpp'), os.path.join(HERE, 'emu', 'emu_raycast.cpp')] + [os.path.join(CSRC, f) for f in ('camera.inl', 'raycast.inl', 'step_core.inl', 'devbuild.h', 'devmodel.h',
                                                                                               'mjcf.cpp', 'model.h')]
        L = _build(os.path.join(BUILD, 'libcassie_emu_camera.so'), deps, ['g++', '-O1', '-std=c++17', '-fPIC', '-shared', src, os.path.join(CSRC, 'mjcf.cpp')])
        L.emu_new.restype = C.c_void_p
        L.emu_new.argtypes = [C.c_char_p, C.c_int]
        L.emu_free.argtypes = [C.c_void_p]
        L.emu_forward.argtypes = [C.c_void_p]
        L.emu_set.argtypes = [C.c_void_p, C.c_char_p, dp, C.c_int]
        L.emu_get.argtypes = [C.c_void_p, C.c_char_p, dp, C.c_int]
        L.emu_ray_slots.argtypes = [C.c_void_p, ip]
        L.emu_cam_render.argtypes = [C.c_void_p, C.c_int, dp, C.c_int, dp, C.POINTER(C.c_float), C.c_int, C.c_int, dp, dp, C.c_double, C.c_int, C.c_int,
                                     C.c_double, dp, dp]
        L.emu_cam_moving.argtypes = [C.c_void_p, ip]
        _libs['e'] = L
    return _libs['e']


def cameras_fixture():
    """tests/golden/cameras.txt: {(model, camera): (body name, pos, quat, fovy, mode)}"""
    out = {}
    for ln in open(os.path.join(GOLDEN, 'cameras.txt')):
        if ln.startswith('#'):
            continue
        t = ln.split()
        out[(t[0], t[1])] = (t[2], np.array([float(x) for x in t[3:6]]), np.array([float(x) for x in t[6:10]]), float(t[10]), int(t[11]))
    return out


class Moving:
    """the moving collision geoms (host geom ids in device-slot order) placed on the body poses xpos [nbody][3], xquat [nbody][4]"""

    def __init__(self, table, geoms, xpos, xquat):
        t = table
        self.type = np.array([int(t['geom_type'][g]) for g in geoms], dtype=np.int32)
        self.pos, self.R = [], []
        for g in geoms:
            b = int(t['geom_bodyid'][g])
            Rb = quat2mat(xquat[4 * b:4 * b + 4])
            self.pos.append(xpos[3 * b:3 * b + 3] + Rb @ t['geom_pos'][3 * g:3 * g + 3])
            self.R.append(Rb @ quat2mat(t['geom_quat'][4 * g:4 * g + 4]))
        self.pos, self.R = np.array(self.pos).reshape(-1, 3), np.array(self.R).reshape(-1, 3, 3)
        self.size = np.array([t['geom_size'][3 * g:3 * g + 3] for g in geoms]).reshape(-1, 3)


def oracle_poses(name, q):
    """xpos, xquat of every body from the fp64 oracle stepper's forward kinematics at qpos q"""
    o = O.OracleSim(os.path.join(GOLDEN, name + '.omodel'))
    o.arr('qpos')[:] = q[:len(o.arr('qpos'))]
    o.forward()
    xpos, xquat = np.array(o.arr('xpos')), np.array(o.arr('xquat'))
    o.close()
    return xpos, xquat


def camera_world(xpos, xquat, body, pos, quat):
    Rb = quat2mat(xquat[4 * body:4 * body + 4])
    return xpos[3 * body:3 * body + 3] + Rb @ pos, Rb @ quat2mat(quat)


def oracle_render(scene, moving, cpos, cR, fovy, W, H, zfar, hf=None):
    """depth [H][W] and geom [H][W] of the fp64 oracle"""
    L = oracle_lib()
    depth, geom = np.zeros((H, W)), np.zeros((H, W), dtype=np.int32)
    pos, R, size = _d(scene.pos), _d(scene.R), _d(scene.size)
    h = None if hf is None else _d(hf)
    mp, mR, ms = _d(moving.pos), _d(moving.R), _d(moving.size)
    L.oracle_camera(len(scene.slots), scene.type.ctypes.data_as(ip), pos.ctypes.data_as(dp), R.ctypes.data_as(dp), size.ctypes.data_as(dp),
                    None if h is None else h.ctypes.data_as(dp), scene.nrow, scene.ncol, scene.hsize.ctypes.data_as(dp),
                    len(moving.type), moving.type.ctypes.data_as(ip), mp.ctypes.data_as(dp), mR.ctypes.data_as(dp), ms.ctypes.data_as(dp),
                    _d(cpos).ctypes.data_as(dp), _d(cR).ctypes.data_as(dp), float(fovy), W, H, float(zfar), depth.ctypes.data_as(dp), geom.ctypes.data_as(ip))
    return depth, geom


def ambiguous(scene, moving, cpos, cR, fovy, W, H, zfar, hf=None, nudge=1e-5):
    """pixels whose hit / miss or geom changes in the oracle when the camera moves by +-nudge in x or y"""
    _, base = oracle_render(scene, moving, cpos, cR, fovy, W, H, zfar, hf)
    amb = np.zeros((H, W), dtype=bool)
    for ax in (0, 1):
        for s in (-nudge, nudge):
            p = _d(cpos).copy()
            p[ax] += s
            amb |= oracle_render(scene, moving, p, cR, fovy, W, H, zfar, hf)[1] != base
    return amb


class EmuCam:
    """one emulated simulator with the camera source"""

    def __init__(self, name, fp32=False):
        self.L = emu_lib()
        self.h = self.L.emu_new(os.path.join(MODELS, name + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h
        self.name = name
        self.table = RS.load_table(os.path.join(MODELS, name + '.cmodel'))
        slots, mov = (C.c_int * 16)(), (C.c_int * 16)()
        ns, nm = self.L.emu_ray_slots(self.h, slots), self.L.emu_cam_moving(self.h, mov)
        self.slots, self.moving_geoms = list(slots)[:ns], list(mov)[:nm]

    def close(self):
        if self.h:
            self.L.emu_free(self.h)
            self.h = None

    def scene(self):
        return RS.Scene(self.name, self.slots)

    def body(self, name):
        return self.table['names_body'].index(name)

    def set_qpos(self, q):
        a = _d(q)
        self.L.emu_set(self.h, b'qpos', a.ctypes.data_as(dp), a.size)
        self.L.emu_forward(self.h)

    def render(self, body, pos, quat, fovy, W, H, zfar, n=1, qpos=None, genv=None, bank=None, poses=False):
        out, st = np.zeros((n, H, W)), np.zeros(7 * 32 + 12 + 256)
        q = None if qpos is None else _d(qpos)
        g = None if genv is None else _d(genv)
        b = None if bank is None else np.ascontiguousarray(bank, dtype=np.float32)
        rc = self.L.emu_cam_render(self.h, n, None if q is None else q.ctypes.data_as(dp), 0 if q is None else q.shape[1],
                                   None if g is None else g.ctypes.data_as(dp), None if b is None else b.ctypes.data_as(C.POINTER(C.c_float)),
                                   0 if b is None else len(b), int(body), _d(pos).ctypes.data_as(dp), _d(quat).ctypes.data_as(dp), float(fovy), W, H, float(zfar),
                                   out.ctypes.data_as(dp), st.ctypes.data_as(dp))
        if rc != 0:
            return None
        return (out, st) if poses else out
