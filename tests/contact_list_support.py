"""The contact lists (cassie_batch_enable_contacts) restated in numpy over the fp64 oracle: MuJoCo's d->contact as the oracle lists it (contacts()),
mj_contactForce decoded from the oracle's efc_force, and the friction of each pair mixed from the model table (mj_contactParam: the geom of higher
priority gives its value, else the larger).  The oracle itself is unchanged.  Also the ctypes wrapper of the emulated F_CL source
(tests/emu/emu_contacts.cpp), built into its own library."""
import ctypes as C
import os
import subprocess

import numpy as np

from conftest import GOLDEN, REPO

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
CON_HEAD, CON_SLOT, CON_MAX, CON_W = 8, 24, 12, 296   # include/cassie_b200.h CASSIE_CON_*
GEOM1, GEOM2, DIM, DIST, POS, FRAME, FORCE, MU, EFC = 0, 1, 2, 3, 4, 7, 16, 22, 23
_LIB = None


def table(model):
    """the oracle's model table of a golden model: name -> list of strings"""
    return {ln.split()[0]: ln.split()[3:] for ln in open(os.path.join(GOLDEN, model + '.omodel')).read().split('\n') if ln.strip()}


def pair_mu(t, g1, g2, friction=None):
    """sliding friction of a geom pair; friction: per-geom sliding coefficients [ngeom] replacing the table's"""
    pr = [int(x) for x in t['geom_priority']]
    f = np.array(t['geom_friction'], float)[0::3] if friction is None else friction
    if pr[g1] != pr[g2]:
        return f[g1] if pr[g1] > pr[g2] else f[g2]
    return max(f[g1], f[g2])


def restate(o, t, friction=None, found=None):
    """the contact-list row [CON_W] of the oracle's current contacts: slots from contacts(), efc addresses ne + nl + the rows of the contacts before,
    forces decoded from efc_force (normal = sum of the pyramid rows, tangent i = (f(2i) - f(2i+1)) mu); found: contacts found (default: listed)"""
    cons = o.contacts()
    f = o.arr('efc_force').copy()
    row = np.zeros(CON_W)
    row[0], row[1] = len(cons), len(cons) if found is None else found
    row[2] = row[1] - row[0]
    r = o.get_int('ne') + o.get_int('nl')
    for k in range(CON_MAX):
        s = row[CON_HEAD + CON_SLOT * k:CON_HEAD + CON_SLOT * (k + 1)]
        if k >= len(cons):
            s[GEOM1] = s[GEOM2] = -1
            continue
        c = cons[k]
        mu = pair_mu(t, c['geom1'], c['geom2'], friction)
        s[GEOM1], s[GEOM2], s[DIM], s[DIST] = c['geom1'], c['geom2'], c['dim'], c['dist']
        s[POS:POS + 3] = c['pos']
        s[FRAME:FRAME + 9] = c['frame'].reshape(9)
        if c['dim'] == 1:
            s[FORCE] = f[r]
            n = 1
        else:
            n = 2 * (c['dim'] - 1)
            p = f[r:r + n]
            s[FORCE] = p.sum()
            for i in range(c['dim'] - 1):
                s[FORCE + 1 + i] = (p[2 * i] - p[2 * i + 1]) * mu
        s[MU], s[EFC] = mu, r
        r += n
    return row


def slots(row):
    return np.asarray(row)[CON_HEAD:].reshape(CON_MAX, CON_SLOT)


def world_forces(row):
    """[listed][3] frame' force[:3]: the force on geom2 in the world frame"""
    s = slots(row)[:int(row[0])]
    return np.einsum('cji,cj->ci', s[:, FRAME:FRAME + 9].reshape(-1, 3, 3), s[:, FORCE:FORCE + 3])


def compare(got, want):
    """(exact fields equal, geometry error relative to its scale, force error relative to the largest force)"""
    g, w = slots(got), slots(want)
    exact = np.array_equal(got[:CON_HEAD], want[:CON_HEAD]) and np.array_equal(g[:, [GEOM1, GEOM2, DIM, EFC]], w[:, [GEOM1, GEOM2, DIM, EFC]])
    geo = [POS, POS + 1, POS + 2] + list(range(FRAME, FRAME + 9)) + [DIST]
    scale = max(1.0, np.abs(w[:, geo]).max())
    geo_err = np.abs(g[:, geo] - w[:, geo]).max() / scale
    fscale = max(1.0, np.abs(w[:, FORCE:FORCE + 6]).max())
    force_err = max(np.abs(g[:, FORCE:FORCE + 6] - w[:, FORCE:FORCE + 6]).max(), np.abs(g[:, MU] - w[:, MU]).max() * fscale) / fscale
    return exact, geo_err, force_err


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_contacts.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_contacts.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci, ip = C.c_void_p, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_int)
        L.emu_cl_new.restype = vp
        L.emu_cl_new.argtypes = [C.c_char_p, ci]
        L.emu_cl_free.argtypes = [vp]
        L.emu_cl_set_frames.argtypes = [vp, C.POINTER(C.c_char_p), ip, ci]
        L.emu_cl_listed.argtypes = [vp, ci]
        L.emu_cl_rows_set.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_cl_step.argtypes = [vp, dp, ci]
        L.emu_cl_mode.argtypes = [vp, ci]
        L.emu_cl_row.argtypes = [vp, dp]
        L.emu_cl_frames.argtypes = [vp, dp]
        L.emu_cl_set_xws.argtypes = [vp, dp]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_model_set.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set_geom.argtypes = [vp, ci, dp, dp, dp]
        L.emu_geom_id.argtypes = [vp, C.c_char_p]
        _LIB = L
    return _LIB


def _dp(a):
    return a.ctypes.data_as(C.POINTER(C.c_double))


class ListSim:
    """one emulated environment on the contact-list twin's source (listed=False: the chain twin's), with optional frames"""

    def __init__(self, model, fp32=False, frames=None):
        self.L = lib()
        self.h = self.L.emu_cl_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model
        self.nfr = 0
        if frames:
            names, kinds = frames
            arr = (C.c_char_p * len(names))(*[n.encode() for n in names])
            assert self.L.emu_cl_set_frames(self.h, arr, (C.c_int * len(kinds))(*kinds), len(names)) == 0
            self.nfr = len(names)

    def close(self):
        if self.h:
            self.L.emu_cl_free(self.h)
            self.h = None

    def listed(self, on):
        self.L.emu_cl_listed(self.h, 1 if on else 0)

    def rows_set(self, what, values):
        a = np.ascontiguousarray(values, dtype=np.float64)
        assert self.L.emu_cl_rows_set(self.h, what.encode(), _dp(a), a.size) == 0, what

    def model_set(self, what, values):
        a = np.ascontiguousarray(values, dtype=np.float64)
        assert self.L.emu_model_set(self.h, what.encode(), _dp(a), a.size) == 0, what

    def set_geom(self, name, pos=None, size=None):
        g = self.L.emu_geom_id(self.h, name.encode())
        arrs = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in (pos, None, size)]
        assert self.L.emu_set_geom(self.h, g, *[None if a is None else _dp(a) for a in arrs]) == 0, name

    def step(self, row, nticks=1):
        self.L.emu_cl_step(self.h, _dp(np.ascontiguousarray(row, dtype=np.float64)), nticks)

    def mode(self, mode):
        self.L.emu_cl_mode(self.h, mode)

    def forward(self):
        self.mode(1)

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), _dp(buf), n)
        assert k >= 0, name
        return buf[:k]

    def set(self, name, arr):
        a = np.ascontiguousarray(arr, dtype=np.float64)
        assert self.L.emu_set(self.h, name.encode(), _dp(a), a.size) >= 0, name

    def place(self, q, v, ws):
        """the state (qpos, qvel, warm start) of an oracle"""
        nq = len(q)
        self.set('qpos', np.r_[q, np.zeros(len(self.get('qpos')) - nq)])
        self.set('qvel', v[:32])
        self.set('qacc_ws', ws[:32])
        if len(v) > 32:
            self.set('xqvel', v[32:])
            x = np.ascontiguousarray(ws[32:], dtype=np.float64)
            self.L.emu_cl_set_xws(self.h, _dp(x))

    def row(self):
        buf = np.zeros(CON_W)
        self.L.emu_cl_row(self.h, _dp(buf))
        return buf

    def frames(self):
        buf = np.zeros(64 * 20)
        return buf[:self.L.emu_cl_frames(self.h, _dp(buf))]
