"""Shared pieces of the inverse-kinematics tests: the TEST-ONLY host emulation of csrc/ik.inl (tests/emu/emu_ik.cpp), the target lists and target rows
both the CPU and the GPU tests solve for, and the fp64 oracle's view of a result (frame poses from its xpos / xquat and the model's sites, frame
velocities from its cvel, Jacobians from its cdof, connect rows from its efc rows)."""
import ctypes as C
import os

import numpy as np

import loops_support as LS
from raycast_support import BUILD, _build
from emu_harness import CSRC, HERE

MODEL_NAMES = LS.MODEL_NAMES
IK_MAX, IK_TW, IK_SLOT = 4, 16, 8
TOL = {False: 1e-10, True: 1e-5}               # the Python defaults of CassieBatch.solve_ik (metres and radians)
LOOP_TOL = {False: 1e-12, True: 1e-6}          # close_loops' defaults: the loops are re-closed to these
WORLD, ROOT = 0, 1
FOOT_W = [1, 1, 1, 0, 1, 1]                    # position, and the orientation about the foot frame's y and z axes (z: the foot's pitch axis)
dp = C.POINTER(C.c_double)
ip = C.POINTER(C.c_int)
_lib = {}


def emu_lib():
    if 'e' not in _lib:
        src = os.path.join(HERE, 'emu', 'emu_ik.cpp')
        deps = [src, os.path.join(HERE, 'emu', 'emu.cpp')] + [os.path.join(CSRC, f) for f in ('ik.inl', 'loops.inl', 'raycast.inl', 'step_core.inl', 'devbuild.h', 'devmodel.h', 'mjcf.cpp', 'model.h')]
        L = _build(os.path.join(BUILD, 'libcassie_emu_ik.so'), deps, ['g++', '-O1', '-std=c++17', '-fPIC', '-shared', src, os.path.join(CSRC, 'mjcf.cpp')])
        L.emu_new.restype = C.c_void_p
        L.emu_new.argtypes = [C.c_char_p, C.c_int]
        L.emu_free.argtypes = [C.c_void_p]
        L.emu_solve_ik.argtypes = [C.c_void_p, C.c_int, dp, dp, C.c_void_p, dp, C.c_int, ip, ip, dp, dp, dp, dp, C.c_int, C.c_double, C.c_double, C.c_int, dp]
        L.emu_ik_columns.argtypes = [C.c_void_p, ip, ip, dp, dp]
        _lib['e'] = L
    return _lib['e']


def feet(model, frame=ROOT):
    """the two foot targets of a model: the foot-pt sites where the model has them, else the foot bodies; position plus the foot's pitch and yaw"""
    t = LS.table(model)
    sites, bodies = list(t['names_site']), list(t['names_body'])
    out = []
    for s in ('left-', 'right-'):
        if s + 'foot-pt' in sites:
            i = sites.index(s + 'foot-pt')
            out.append(dict(name=s + 'foot-pt', kind=1, body=int(t['site_bodyid'][i]), pos=t['site_pos'][3 * i:3 * i + 3].copy(), quat=t['site_quat'][4 * i:4 * i + 4].copy(), frame=frame, w=list(FOOT_W)))
        else:
            out.append(dict(name=s + 'foot', kind=0, body=bodies.index(s + 'foot'), pos=np.zeros(3), quat=np.array([1.0, 0, 0, 0]), frame=frame, w=list(FOOT_W)))
    return out


class EmuIk:
    """the inverse-kinematics source on the host, for one model and precision"""

    def __init__(self, model, fp32):
        self.L = emu_lib()
        self.h = self.L.emu_new(os.path.join(LS.MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model
        self.fp32 = fp32

    def solve(self, qpos, qvel, spec, targets, mask=None, bpos=None, max_iter=100, tol=None, velocities=0, status=None):
        """solves copies of qpos [n][nq] / qvel [n][nv] for the target rows [n][IK_MAX][IK_TW]; returns (qpos, qvel, status [n][8], selected count)"""
        q, v = np.array(qpos, dtype=np.float64), np.array(qvel, dtype=np.float64)
        n, nt = q.shape[0], len(spec)
        st = np.zeros((n, IK_SLOT)) if status is None else np.array(status, dtype=np.float64)
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        b = None if bpos is None else np.ascontiguousarray(bpos, dtype=np.float64)
        body = np.array([s['body'] for s in spec] + [0], dtype=np.int32)
        frame = np.array([s['frame'] for s in spec] + [0], dtype=np.int32)
        fpos = np.concatenate([np.ravel(s['pos']) for s in spec] + [np.zeros(3)])
        fquat = np.concatenate([np.ravel(s['quat']) for s in spec] + [np.zeros(4)])
        w = np.concatenate([np.ravel(np.asarray(s['w'], dtype=np.float64)) for s in spec] + [np.zeros(6)])
        tg = np.ascontiguousarray(targets, dtype=np.float64).reshape(n, IK_MAX, IK_TW)
        k = self.L.emu_solve_ik(self.h, n, q.ctypes.data_as(dp), v.ctypes.data_as(dp), None if m is None else m.ctypes.data, None if b is None else b.ctypes.data_as(dp),
                                nt, body.ctypes.data_as(ip), frame.ctypes.data_as(ip), fpos.ctypes.data_as(dp), fquat.ctypes.data_as(dp), w.ctypes.data_as(dp),
                                tg.ctypes.data_as(dp), int(max_iter), float(TOL[self.fp32] if tol is None else tol), float(LOOP_TOL[self.fp32]), int(velocities),
                                st.ctypes.data_as(dp))
        return q, v, st, k

    def columns(self):
        """the free columns: dof, limited, lo, hi (arrays over the columns)"""
        dof, lim = np.zeros(32, dtype=np.int32), np.zeros(32, dtype=np.int32)
        lo, hi = np.zeros(32), np.zeros(32)
        nc = self.L.emu_ik_columns(self.h, dof.ctypes.data_as(ip), lim.ctypes.data_as(ip), lo.ctypes.data_as(dp), hi.ctypes.data_as(dp))
        assert nc > 0
        return dof[:nc], lim[:nc].astype(bool), lo[:nc], hi[:nc]

    def __del__(self):
        if getattr(self, 'h', None):
            self.L.emu_free(self.h)
            self.h = None


def _q2m(q):
    return LS._q2m(q)


def _qmul(a, b):
    return LS._qmul(a, b)


def _conj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def rotvec(q):
    """rotation vector of a unit quaternion, the short way round"""
    q = np.asarray(q, dtype=np.float64) / np.linalg.norm(q)
    if q[0] < 0:
        q = -q
    s = np.linalg.norm(q[1:])
    return q[1:] * (2 * np.arctan2(s, q[0]) / s if s > 0 else 2.0)


def dlog(e):
    """J_l^-1(e): the rate of the rotation vector e under a left perturbation"""
    th = np.linalg.norm(e)
    c = 1 / 12 + th * th / 720 if th < 1e-4 else 1 / th ** 2 - (1 + np.cos(th)) / (2 * th * np.sin(th))
    E = np.array([[0, -e[2], e[1]], [e[2], 0, -e[0]], [-e[1], e[0], 0]])
    return np.eye(3) - 0.5 * E + c * E @ E


class OracleFrames:
    """the fp64 oracle's view of target frames: pose and velocity in the target's expression frame, and the Jacobians of the position and of the
    rotation-vector error over every dof, from xpos / xquat / xmat, cvel and cdof (MuJoCo's mj_jac), and the connect rows efc_pos / efc_J"""

    def __init__(self, model):
        self.t = LS.table(model)
        self.o = LS.oracle(model)
        self.neq3 = 3 * int(self.t['neq'][0])
        self.bp0 = self.o.model_arr('body_pos').copy()
        self.nv = self.o.nv
        t = self.t
        self.root = list(t['names_body']).index('cassie-pelvis')   # the root body: the pelvis
        par = t['body_parentid'].astype(int)
        self.dofs = []   # dofs that move each body
        for b in range(int(t['nbody'][0])):
            ds, p = [], b
            while p > 0:
                a, k = int(t['body_dofadr'][p]), int(t['body_dofnum'][p])
                ds += list(range(a, a + k)) if k and a >= 0 else []
                p = par[p]
            self.dofs.append(sorted(ds))

    def set(self, qpos, qvel=None, bpos=None):
        self.o.model_arr('body_pos')[:] = self.bp0 if bpos is None else np.ravel(bpos)
        self.o.arr('qpos')[:] = qpos
        self.o.arr('qvel')[:] = 0 if qvel is None else qvel
        self.o.forward()

    def _world(self, s):
        b = s['body']
        xp, xq, xm = self.o.arr('xpos').reshape(-1, 3)[b], self.o.arr('xquat').reshape(-1, 4)[b], self.o.arr('xmat').reshape(-1, 3, 3)[b]
        return xp + xm @ np.asarray(s['pos']), _qmul(xq, np.asarray(s['quat']) / np.linalg.norm(s['quat']))

    def pose(self, s):
        """position and quaternion of target s's frame in its expression frame (after set)"""
        p, q = self._world(s)
        if s['frame'] == ROOT:
            r = self.root
            pr, qr, Rr = self.o.arr('xpos').reshape(-1, 3)[r], self.o.arr('xquat').reshape(-1, 4)[r], self.o.arr('xmat').reshape(-1, 3, 3)[r]
            p, q = Rr.T @ (p - pr), _qmul(_conj(qr), q)
        return p, q / np.linalg.norm(q)

    def jacobian(self, s):
        """world jacp [3][nv], jacr [3][nv] of target s's frame point (root dofs zeroed for a root target), and the expression frame's rotation"""
        p, _ = self._world(s)
        cdof = self.o.arr('cdof').reshape(-1, 6)
        com = self.o.arr('subtree_com').reshape(-1, 3)[self.root]
        jp, jr = np.zeros((3, self.nv)), np.zeros((3, self.nv))
        for d in self.dofs[s['body']]:
            if s['frame'] == ROOT and d in self.dofs[self.root]:
                continue
            jr[:, d] = cdof[d, :3]
            jp[:, d] = cdof[d, 3:] + np.cross(cdof[d, :3], p - com)
        Re = self.o.arr('xmat').reshape(-1, 3, 3)[self.root] if s['frame'] == ROOT else np.eye(3)
        return jp, jr, Re

    def velocity(self, s, qvel):
        """linear and angular velocity of target s's frame in its expression frame (relative to the root body for a root target)"""
        jp, jr, Re = self.jacobian(s)
        return Re.T @ (jp @ qvel), Re.T @ (jr @ qvel)

    def rows(self, s, row):
        """target s's position error [3] and rotation vector [3] against a target row (after set)"""
        p, q = self.pose(s)
        tq = np.asarray(row[3:7]) / np.linalg.norm(row[3:7])
        return p - row[:3], rotvec(_qmul(_conj(tq), q))

    def connect(self):
        return self.o.arr('efc_pos')[:self.neq3].copy(), self.o.efc_J()[:self.neq3]


def residuals(model, spec, q, targets, bpos=None):
    """per state: max weighted-row position error, max weighted-row orientation error, max connect residual (fp64 oracle)"""
    F = OracleFrames(model)
    out = []
    for i in range(len(q)):
        F.set(q[i], None, None if bpos is None else bpos[i])
        pe, oe = 0.0, 0.0
        for k, s in enumerate(spec):
            dpos, e = F.rows(s, targets[i, k])
            w = np.asarray(s['w'])
            pe = max(pe, np.abs(dpos[w[:3] != 0]).max(initial=0))
            oe = max(oe, np.abs(e[w[3:] != 0]).max(initial=0))
        r, _ = F.connect()
        out.append((pe, oe, np.abs(r).max(initial=0)))
    return np.array(out)


def objective(F, spec, row_set):
    """sum over the targets of |w e|^2 at the oracle's current state"""
    f = 0.0
    for k, s in enumerate(spec):
        dpos, e = F.rows(s, row_set[k])
        f += float(np.sum((np.asarray(s['w'][:3]) * dpos) ** 2) + np.sum((np.asarray(s['w'][3:]) * e) ** 2))
    return f


def gradient(F, spec, row_set):
    """the gradient of the objective over every dof (the position rows' jacp, the orientation rows' J_l^-1 R_t' R_e' jacr), at the current state"""
    g = np.zeros(F.nv)
    for k, s in enumerate(spec):
        dpos, e = F.rows(s, row_set[k])
        jp, jr, Re = F.jacobian(s)
        tq = np.asarray(row_set[k][3:7]) / np.linalg.norm(row_set[k][3:7])
        w = np.asarray(s['w'], dtype=np.float64)
        g += 2 * (Re.T @ jp).T @ (w[:3] ** 2 * dpos)
        g += 2 * (dlog(e) @ _q2m(tq).T @ Re.T @ jr).T @ (w[3:] ** 2 * e)
    return g


MOTOR_JOINTS = [s + j for s in ('left-', 'right-') for j in ('hip-roll', 'hip-yaw', 'hip-pitch', 'knee', 'foot')]


def motor_qpos(model):
    t = LS.table(model)
    names = list(t['names_joint'])
    return np.array([int(t['jnt_qposadr'][names.index(j)]) for j in MOTOR_JOINTS])


def motor_range(model):
    t = LS.table(model)
    names = list(t['names_joint'])
    return np.array([t['jnt_range'][2 * names.index(j):2 * names.index(j) + 2] for j in MOTOR_JOINTS])


def target_rows(model, spec, q, qvel=None, bpos=None):
    """target rows [n][IK_MAX][IK_TW] from the oracle's frames at states q (and velocities qvel, else zero)"""
    F = OracleFrames(model)
    out = np.zeros((len(q), IK_MAX, IK_TW))
    for i in range(len(q)):
        F.set(q[i], None if qvel is None else qvel[i], None if bpos is None else bpos[i])
        for k, s in enumerate(spec):
            p, qq = F.pose(s)
            out[i, k, :3], out[i, k, 3:7] = p, qq
            if qvel is not None:
                v, w = F.velocity(s, qvel[i])
                out[i, k, 7:10], out[i, k, 10:13] = v, w
    return out


def reachable(model, n, seed, spread=0.3, fp32=False):
    """n poses closed from random in-range motor angles (the standing motors plus U(-spread, spread), clipped to their ranges) by close_loops' source in
    fp64, and the standing start pose they are solved from: (start qpos [n][nq], posed qpos [n][nq])"""
    rng = np.random.default_rng(seed)
    q0 = LS.standing(model)
    mq, mr = motor_qpos(model), motor_range(model)
    q = np.tile(q0, (n, 1))
    q[:, mq] = np.clip(q[:, mq] + rng.uniform(-spread, spread, (n, len(mq))), mr[:, 0], mr[:, 1])
    t = LS.table(model)
    qc, _, st, _ = LS.EmuLoops(model, False).close(q, np.zeros((n, int(t['nv'][0]))), max_iter=50, tol=1e-13)
    assert (st[:, 1] >= 0).all()
    start = np.tile(q0, (n, 1))
    if fp32:
        start = start.astype(np.float32).astype(np.float64)
    return start, qc
