"""Shared pieces of the camera-set tests (several cameras per launch, per-environment mounts, geom ids): the host emulation of the camera-set source
(csrc/camera_set.inl in tests/emu/emu_cameras.cpp, its own library), the three-camera rig the tests use, and the oracle's view of one camera of one environment."""
import ctypes as C
import os

import numpy as np

import camera_support as CS
from emu_harness import CSRC, HERE
from raycast_support import BUILD, _build, _d, dp, quat2mat

ip = C.POINTER(C.c_int)
_libs = {}
SLOT = 8   # CASSIE_CAMENV_SLOT: pos[3], quat[4], fovy in degrees


def emu_lib():
    if 'e' not in _libs:
        src = os.path.join(HERE, 'emu', 'emu_cameras.cpp')
        deps = [src, os.path.join(HERE, 'emu', 'emu.cpp'), os.path.join(HERE, 'emu', 'emu_raycast.cpp')] + [
            os.path.join(CSRC, f) for f in ('camera_set.inl', 'camera.inl', 'raycast.inl', 'step_core.inl', 'devbuild.h', 'devmodel.h', 'mjcf.cpp', 'model.h')]
        L = _build(os.path.join(BUILD, 'libcassie_emu_cameras.so'), deps, ['g++', '-O1', '-std=c++17', '-fPIC', '-shared', src, os.path.join(CSRC, 'mjcf.cpp')])
        L.emu_new.restype = C.c_void_p
        L.emu_new.argtypes = [C.c_char_p, C.c_int]
        L.emu_free.argtypes = [C.c_void_p]
        L.emu_ray_slots.argtypes = [C.c_void_p, ip]
        L.emu_cams_render.argtypes = [C.c_void_p, C.c_int, dp, C.c_int, dp, C.POINTER(C.c_float), C.c_int, C.c_int, ip, dp, dp, dp, C.c_int, C.c_int,
                                      C.c_double, dp, dp, ip]
        _libs['e'] = L
    return _libs['e']


class EmuCams(CS.EmuCam):
    """one emulated simulator with the camera source, rendering camera sets"""

    def __init__(self, name, fp32=False):
        super().__init__(name, fp32)
        self.S = emu_lib()
        self.hs = self.S.emu_new(os.path.join(CS.MODELS, name + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.hs

    def close(self):
        super().close()
        if self.hs:
            self.S.emu_free(self.hs)
            self.hs = None

    def render_set(self, cams, W, H, zfar, n, qpos=None, genv=None, bank=None, cenv=None, geoms=False):
        """cams: [(body id, pos, quat, fovy)]; cenv [n][k][SLOT] or None.  depth [n][k][H][W] (and geom ids), or None for a refused set"""
        k = len(cams)
        body = np.array([c[0] for c in cams], dtype=np.int32)
        pos, quat, fovy = (_d([np.asarray(c[i], float) for c in cams]) for i in (1, 2, 3))
        out, gid = np.zeros((n, k, H, W)), np.zeros((n, k, H, W), dtype=np.int32)
        q = None if qpos is None else _d(qpos)
        g = None if genv is None else _d(genv)
        b = None if bank is None else np.ascontiguousarray(bank, dtype=np.float32)
        ce = None if cenv is None else _d(cenv)
        rc = self.S.emu_cams_render(self.hs, n, None if q is None else q.ctypes.data_as(dp), 0 if q is None else q.shape[1],
                                    None if g is None else g.ctypes.data_as(dp), None if b is None else b.ctypes.data_as(C.POINTER(C.c_float)),
                                    0 if b is None else len(b), k, body.ctypes.data_as(ip), pos.ctypes.data_as(dp), quat.ctypes.data_as(dp),
                                    fovy.ctypes.data_as(dp), W, H, float(zfar), None if ce is None else ce.ctypes.data_as(dp), out.ctypes.data_as(dp),
                                    gid.ctypes.data_as(ip) if geoms else None)
        if rc != 0:
            return None
        return (out, gid) if geoms else out

    def model_geom(self, g):
        """the oracle's geom numbering (static slot g, moving geom 100 + m, -1) in the model's"""
        g = np.asarray(g)
        st = np.array(self.slots + [-1])[np.clip(g, 0, len(self.slots))]
        mv = np.array(self.moving_geoms + [-1])[np.clip(g - 100, 0, len(self.moving_geoms))]
        return np.where(g < 0, -1, np.where(g >= 100, mv, st))


def mat2quat(R):
    w = np.sqrt(max(0.0, 1 + R[0, 0] + R[1, 1] + R[2, 2])) / 2
    if w > 1e-3:
        return np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])
    i = int(np.argmax(np.diag(R)))
    j, k = (i + 1) % 3, (i + 2) % 3
    v = np.zeros(4)
    v[1 + i] = np.sqrt(max(0.0, 1 + R[i, i] - R[j, j] - R[k, k])) / 2
    v[0] = (R[k, j] - R[j, k]) / (4 * v[1 + i])
    v[1 + j] = (R[j, i] + R[i, j]) / (4 * v[1 + i])
    v[1 + k] = (R[k, i] + R[i, k]) / (4 * v[1 + i])
    return v


def look_at(eye, target, up=(0, 0, 1)):
    z = np.asarray(eye, float) - target
    z /= np.linalg.norm(z)
    x = np.cross(up, z)
    x /= np.linalg.norm(x)
    return np.stack([x, np.cross(z, x), z], 1)


def rig(model, body_of, q0):
    """the three cameras of the tests: the egocentric mount of cassie_depth.xml on the pelvis, a camera 0.1 m along the left tarsus looking straight
    down at the standing state q0, and a world-body camera 2.5 m away looking at the robot"""
    _, pos, quat, fovy, _ = CS.cameras_fixture()[('cassie_depth', 'egocentric')]
    tar = body_of('left-tarsus')
    xpos, xquat = CS.oracle_poses(model, q0)
    Rt = quat2mat(xquat[4 * tar:4 * tar + 4])
    down = np.diag([1.0, -1.0, -1.0])   # camera -z along world -z
    eye = np.array([2.2, -1.2, 1.4])
    return [(body_of('cassie-pelvis'), pos, quat, fovy), (tar, np.array([0.1, 0.0, 0.0]), mat2quat(Rt.T @ down), 80.0),
            (0, eye, mat2quat(look_at(eye, [0.0, 0.0, 0.6])), 55.0)]


def random_rows(rng, cams, n):
    """per-environment mount rows [n][k][SLOT]: each camera's pos moved by up to 2 cm, turned by up to 3 degrees, fovy changed by up to 5 degrees"""
    k = len(cams)
    rows = np.zeros((n, k, SLOT))
    for e in range(n):
        for c, (_, pos, quat, fovy) in enumerate(cams):
            ax = rng.normal(size=3)
            ang = np.radians(rng.uniform(-3, 3))
            dq = np.concatenate([[np.cos(ang / 2)], np.sin(ang / 2) * ax / np.linalg.norm(ax)])
            q = np.asarray(quat, float) / np.linalg.norm(quat)
            rows[e, c, 0:3] = np.asarray(pos, float) + rng.uniform(-0.02, 0.02, 3)
            rows[e, c, 3:7] = quat_mul(q, dq) * rng.uniform(0.5, 2.0)   # not unit: the kernel normalises
            rows[e, c, 7] = fovy + rng.uniform(-5, 5)
    return rows


def quat_mul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def oracle_view(table, moving_geoms, model, q, scene, body, pos, quat, fovy, W, H, zfar, hf=None, amb=False):
    """the oracle's depth and geom (its own numbering) of one camera (pos / quat in the body frame) at qpos q, and optionally its ambiguous pixels"""
    xpos, xquat = CS.oracle_poses(model, q)
    mv = CS.Moving(table, moving_geoms, xpos, xquat)
    cpos, cR = CS.camera_world(xpos, xquat, body, np.asarray(pos, float), np.asarray(quat, float) / np.linalg.norm(quat))
    d, g = CS.oracle_render(scene, mv, cpos, cR, fovy, W, H, zfar, hf)
    return (d, g, CS.ambiguous(scene, mv, cpos, cR, fovy, W, H, zfar, hf) if amb else None)
