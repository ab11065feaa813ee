"""Shared pieces of the loop-closure tests: the TEST-ONLY host emulation of csrc/loops.inl (tests/emu/emu_loops.cpp), the start states both the CPU and
the GPU tests close, and the fp64 oracle's view of a result (its connect rows efc_pos / efc_J at the closed state)."""
import ctypes as C
import os

import numpy as np

import oracle as O
from raycast_support import BUILD, GOLDEN, MODELS, _build, load_table
from emu_harness import CSRC, HERE

MODEL_NAMES = ('cassie', 'cassie_mass', 'cassie_hfield', 'cassie_tray_box')
LAMBDA = {False: 1e-10, True: 1e-6}          # the kernel's damping per precision (fp32: True)
STAND = dict(pTarget=[0.0045, 0, 0.4973, -1.1997, -1.5968] * 2, pGain=[70, 70, 100, 100, 50] * 2, dGain=[7, 7, 8, 8, 5] * 2)
dp = C.POINTER(C.c_double)
_lib = {}


def emu_lib():
    if 'e' not in _lib:
        src = os.path.join(HERE, 'emu', 'emu_loops.cpp')
        deps = [src, os.path.join(HERE, 'emu', 'emu.cpp'), os.path.join(CSRC, 'loops.inl'), os.path.join(CSRC, 'raycast.inl'), os.path.join(CSRC, 'step_core.inl'),
                os.path.join(CSRC, 'devbuild.h'), os.path.join(CSRC, 'devmodel.h'), os.path.join(CSRC, 'mjcf.cpp'), os.path.join(CSRC, 'model.h')]
        L = _build(os.path.join(BUILD, 'libcassie_emu_loops.so'), deps, ['g++', '-O1', '-std=c++17', '-fPIC', '-shared', src, os.path.join(CSRC, 'mjcf.cpp')])
        L.emu_new.restype = C.c_void_p
        L.emu_new.argtypes = [C.c_char_p, C.c_int]
        L.emu_free.argtypes = [C.c_void_p]
        L.emu_close_loops.argtypes = [C.c_void_p, C.c_int, dp, dp, C.c_void_p, dp, C.c_int, C.c_double, dp]
        L.emu_loop_free.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
        _lib['e'] = L
    return _lib['e']


class EmuLoops:
    """the loop-closure source on the host, for one model and precision"""

    def __init__(self, model, fp32):
        self.L = emu_lib()
        self.h = self.L.emu_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model
        self.fp32 = fp32

    def close(self, qpos, qvel, mask=None, bpos=None, max_iter=20, tol=1e-12, status=None):
        """closes copies of qpos [n][nq] / qvel [n][nv]; returns (qpos, qvel, status [n][4], selected count)"""
        q, v = np.array(qpos, dtype=np.float64), np.array(qvel, dtype=np.float64)
        n = q.shape[0]
        st = np.zeros((n, 4)) if status is None else np.array(status, dtype=np.float64)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        b = None if bpos is None else np.ascontiguousarray(bpos, dtype=np.float64)
        k = self.L.emu_close_loops(self.h, n, q.ctypes.data_as(dp), v.ctypes.data_as(dp), None if m is None else m.ctypes.data, None if b is None else b.ctypes.data_as(dp),
                                   int(max_iter), float(tol), st.ctypes.data_as(dp))
        return q, v, st, k

    def free(self, nq, nv):
        qf, vf = np.zeros(nq, dtype=np.int32), np.zeros(nv, dtype=np.int32)
        assert self.L.emu_loop_free(self.h, qf.ctypes.data_as(C.POINTER(C.c_int)), vf.ctypes.data_as(C.POINTER(C.c_int))) >= 0
        return qf.astype(bool), vf.astype(bool)

    def __del__(self):
        if getattr(self, 'h', None):
            self.L.emu_free(self.h)
            self.h = None


def table(model):
    return load_table(os.path.join(MODELS, model + '.cmodel'))


def oracle(model):
    return O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))


_standing = {}


def standing(model):
    """a settled standing state: 0.5 s of the standing PD from the initial state of cassie.xml on the fp64 oracle (the heavier cassie_mass crouches
    into poses where noise can open a loop beyond closing), with the model's own initial coordinates beyond the 35 of the Cassie tree"""
    if 'q' not in _standing:
        o = oracle('cassie')
        u = O.make_pd(**STAND)
        for _ in range(1000):
            o.step_pd(u)
        _standing['q'] = o.arr('qpos').copy()
    q = oracle(model).arr('qpos').copy()
    q[:35] = _standing['q']
    return q


def loop_bodies(t):
    """the bodies inside the legs' loops that the offset start states move: achilles rod and heel spring (the spatial loop) and the foot crank, whose
    offset is kept in the plane of the plantar-rod loop"""
    names = list(t['names_body'])
    return [names.index(s + b) for s in ('left-', 'right-') for b in ('achilles-rod', 'heel-spring', 'foot-crank')]


def _q2m(q):
    w, x, y, z = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    return np.array([[w*w+x*x-y*y-z*z, 2*(x*y-w*z), 2*(x*z+w*y)], [2*(x*y+w*z), w*w-x*x+y*y-z*z, 2*(y*z-w*x)], [2*(x*z-w*y), 2*(y*z+w*x), w*w-x*x-y*y+z*z]])


def start_states(model, kind, n, seed, fp32=False):
    """n start states: qpos [n][nq], qvel [n][nv], body offsets [n][nbody][3] or None.  'noisy': the initial state with N(0, 0.05 rad) on every joint
    coordinate beyond the pelvis (rod quaternions left unnormalised); 'standing': a settled standing state with the same noise; 'offsets': the initial
    state under per-environment offsets N(0, 5 mm) of the loop bodies.  qvel: N(0, 0.5) on every main-tree dof.  fp32: rounded to float32 first"""
    rng = np.random.default_rng(seed)
    t = table(model)
    nq, nv, nb = int(t['nq'][0]), int(t['nv'][0]), int(t['nbody'][0])
    nqm, nvm = (35, 32)
    if kind == 'standing':
        q0 = standing(model)
    else:
        o = oracle(model)
        q0 = o.arr('qpos').copy()
    q = np.tile(q0, (n, 1))
    v = np.zeros((n, nv))
    v[:, :nvm] = 0.5 * rng.standard_normal((n, nvm))
    bpos = None
    if kind in ('noisy', 'standing'):
        q[:, 7:nqm] += 0.05 * rng.standard_normal((n, nqm - 7))
    else:
        bpos = np.tile(t['body_pos'].reshape(nb, 3), (n, 1, 1))
        for b in loop_bodies(t):
            d = 0.005 * rng.standard_normal((n, 3))
            if 'foot-crank' in t['names_body'][b]:   # in the plane of the plantar-rod loop: off the crank's hinge axis, in the tarsus frame
                j = int(t['body_jntadr'][b])
                ax = _q2m(t['body_quat'][4 * b:4 * b + 4]) @ t['jnt_axis'][3 * j:3 * j + 3]
                d -= np.outer(d @ ax, ax)
            bpos[:, b] += d
    if fp32:
        q, v = q.astype(np.float32).astype(np.float64), v.astype(np.float32).astype(np.float64)
        bpos = None if bpos is None else bpos.astype(np.float32).astype(np.float64)
    return q, v, bpos


class OracleRows:
    """the fp64 oracle's connect rows at given states: residual efc_pos and Jacobian efc_J of the equality rows"""

    def __init__(self, model):
        self.o = oracle(model)
        self.neq3 = 3 * int(table(model)['neq'][0])
        self.bp0 = self.o.model_arr('body_pos').copy()

    def rows(self, qpos, bpos=None):
        self.o.model_arr('body_pos')[:] = self.bp0 if bpos is None else np.ravel(bpos)
        self.o.arr('qpos')[:] = qpos
        self.o.forward()
        return self.o.arr('efc_pos')[:self.neq3].copy(), self.o.efc_J()[:self.neq3]

    def residuals(self, qpos, qvel, bpos=None):
        """max |p1 - p2| and max |J qvel| of every state"""
        out = []
        for i in range(len(qpos)):
            r, J = self.rows(qpos[i], None if bpos is None else bpos[i])
            out.append((np.abs(r).max(), np.abs(J @ qvel[i]).max()))
        return np.array(out)


def _qmul(a, b):
    return np.array([a[0]*b[0]-a[1]*b[1]-a[2]*b[2]-a[3]*b[3], a[0]*b[1]+a[1]*b[0]+a[2]*b[3]-a[3]*b[2], a[0]*b[2]-a[1]*b[3]+a[2]*b[0]+a[3]*b[1], a[0]*b[3]+a[1]*b[2]-a[2]*b[1]+a[3]*b[0]])


def restate(model, rows, qpos, qvel, vfree, bpos=None, max_iter=20, tol=1e-12, lam=1e-10):
    """numpy restatement of the closure of one state on the oracle's efc rows: returns (qpos, qvel, iterations or -1)"""
    t = table(model)
    q, v = np.array(qpos, dtype=np.float64), np.array(qvel, dtype=np.float64)
    free = np.flatnonzero(vfree)
    joints = [j for j in range(int(t['njnt'][0])) if vfree[int(t['jnt_dofadr'][j])]]
    for j in joints:
        if int(t['jnt_type'][j]) == 1:
            a = int(t['jnt_qposadr'][j]); q[a:a + 4] /= np.linalg.norm(q[a:a + 4])
    it = 0
    while True:
        r, J = rows.rows(q, bpos)
        if np.abs(r).max() <= tol:
            break
        if it == max_iter:
            return np.array(qpos, dtype=np.float64), np.array(qvel, dtype=np.float64), -1
        Jf = J[:, free]
        dq = np.zeros(len(v))
        dq[free] = -Jf.T @ np.linalg.solve(Jf @ Jf.T + lam * np.eye(len(r)), r)
        for j in joints:
            a, d = int(t['jnt_qposadr'][j]), int(t['jnt_dofadr'][j])
            if int(t['jnt_type'][j]) != 1:
                q[a] += dq[d]
                continue
            w = dq[d:d + 3]; ang = np.linalg.norm(w)
            qr = np.array([1.0, 0, 0, 0]) if ang == 0 else np.concatenate([[np.cos(ang / 2)], w / ang * np.sin(ang / 2)])
            q[a:a + 4] = _qmul(q[a:a + 4] / np.linalg.norm(q[a:a + 4]), qr)
        it += 1
    Jf = J[:, free]
    v[free] -= Jf.T @ np.linalg.solve(Jf @ Jf.T + lam * np.eye(len(r)), J @ v)
    return (np.array(qpos, dtype=np.float64) if it == 0 else q), v, it
