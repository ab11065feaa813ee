"""Frame rows (cassie_batch_set_frames): the product's stepper source in the host emulation with a frame table, i.e. the F_FR instance, against the
oracle's kinematics, velocities and contact list.  The GPU twins are in tests/test_gpu_frames.py.

The emulation with a frame row is tests/emu/emu_frames.cpp (emu.cpp plus the row), built into its own library here.  The oracle side restates the
reference queries from the oracle's arrays: xpos / xquat, site_xpos and mju_mat2Quat(site_xmat) (src/cassiemujoco.c:1242-1252, 1543-1553), cvel after
mj_comVel (cassie_sim_body_velocities, :1752-1760) and the contact forces of the bodies (cassie_sim_body_contact_force, :1781-1809)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from test_model_variants import PD_ROW

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
W, POS, QUAT, VEL, CFRC = 20, 0, 3, 7, 13
ZERO_ROW = np.zeros(50)   # no torque, no gains: the robot falls
_LIB = None


def fr_lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_frames.so')
        srcs = [os.path.join(E.HERE, 'emu', 'emu_frames.cpp'), os.path.join(E.CSRC, 'mjcf.cpp'), os.path.join(E.HERE, 'emu', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], srcs[1]])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_fr_new.restype = vp
        L.emu_fr_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_fr_free', 'emu_fr_forward', 'emu_plain'):
            getattr(L, n).argtypes = [vp]
        L.emu_fr_set.argtypes = [vp, C.POINTER(C.c_char_p), C.POINTER(ci), ci]
        L.emu_fr_step.argtypes = [vp, dp, ci]
        L.emu_fr_row.argtypes = [vp, dp]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


class FrameSim:
    """one emulated environment on the extended instance; with frames set the F_FR path runs"""

    def __init__(self, model, fp32=False):
        self.L = fr_lib()
        self.h = self.L.emu_fr_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h, model

    def close(self):
        if self.h:
            self.L.emu_fr_free(self.h)
            self.h = None

    def set_frames(self, names, kinds):
        arr = (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])
        ks = (C.c_int * max(1, len(kinds)))(*kinds)
        return self.L.emu_fr_set(self.h, arr, ks, len(names))

    def plain_aux_off(self):
        self.L.emu_plain(self.h)

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def frames(self):
        buf = np.zeros(64 * W)
        n = self.L.emu_fr_row(self.h, buf.ctypes.data_as(C.POINTER(C.c_double)))
        return buf[:n * W].reshape(n, W)

    def step(self, pd50, nticks=1):
        a = np.ascontiguousarray(pd50, dtype=np.float64)
        self.L.emu_fr_step(self.h, a.ctypes.data_as(C.POINTER(C.c_double)), nticks)

    def forward(self):
        self.L.emu_fr_forward(self.h)


def omodel(model):
    """{key: values} of a golden oracle model table (site and body tables, names)"""
    out = {}
    for ln in open(os.path.join(GOLDEN, model + '.omodel')):
        t = ln.split()
        if len(t) >= 3 and t[1] in ('I', 'F', 'S'):
            v = t[3:]
            out[t[0]] = v if t[1] == 'S' else np.array([float(x) for x in v])
    return out


def all_frames(model):
    m = omodel(model)
    return list(m['names_body']) + list(m['names_site']), [0] * len(m['names_body']) + [1] * len(m['names_site'])


def mul_quat(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat2mat(q):
    w, x, y, z = q
    return np.array([[1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y)], [2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)]])


def mat2quat(R):
    """mju_mat2Quat: MuJoCo's branches, and so its sign"""
    t = R[0, 0] + R[1, 1] + R[2, 2]
    if t > 0:
        s = np.sqrt(t + 1) * 2
        return np.array([0.25 * s, (R[2, 1] - R[1, 2]) / s, (R[0, 2] - R[2, 0]) / s, (R[1, 0] - R[0, 1]) / s])
    if R[0, 0] > R[1, 1] and R[0, 0] > R[2, 2]:
        s = np.sqrt(1 + R[0, 0] - R[1, 1] - R[2, 2]) * 2
        return np.array([(R[2, 1] - R[1, 2]) / s, 0.25 * s, (R[0, 1] + R[1, 0]) / s, (R[0, 2] + R[2, 0]) / s])
    if R[1, 1] > R[2, 2]:
        s = np.sqrt(1 + R[1, 1] - R[0, 0] - R[2, 2]) * 2
        return np.array([(R[0, 2] - R[2, 0]) / s, (R[0, 1] + R[1, 0]) / s, 0.25 * s, (R[1, 2] + R[2, 1]) / s])
    s = np.sqrt(1 + R[2, 2] - R[0, 0] - R[1, 1]) * 2
    return np.array([(R[1, 0] - R[0, 1]) / s, (R[0, 2] + R[2, 0]) / s, (R[1, 2] + R[2, 1]) / s, 0.25 * s])


def contact_world_forces(o, m):
    """[(body1, body2, world force)] of the oracle's contacts: mj_contactForce (pyramid decode) rotated into the world frame"""
    f = o.arr('efc_force')
    adr = o.get_int('ne') + o.get_int('nl')
    gb = m['geom_bodyid'].astype(int)
    fr, pr = m['geom_friction'].reshape(-1, 3), m['geom_priority'].astype(int)
    out = []
    for c in o.contacts():
        g1, g2, dim = c['geom1'], c['geom2'], c['dim']
        if dim == 1:
            loc = np.array([f[adr], 0, 0])
            adr += 1
        else:
            mu = fr[g1, 0] if pr[g1] > pr[g2] else (fr[g2, 0] if pr[g2] > pr[g1] else max(fr[g1, 0], fr[g2, 0]))
            r = f[adr:adr + 4]
            loc = np.array([r.sum(), (r[0] - r[1]) * mu, (r[2] - r[3]) * mu])
            adr += 4
        out.append((gb[g1], gb[g2], c['frame'].T @ loc))
    return out


def oracle_frames(o, m, names, kinds):
    """the reference's query results for every frame after the oracle's last step / forward, in the row layout"""
    nb = len(m['names_body'])
    xpos, xquat, xmat = o.arr('xpos').reshape(-1, 3), o.arr('xquat').reshape(-1, 4), o.arr('xmat').reshape(-1, 3, 3)
    o.L.osim_comvel(o.h)
    cvel = o.arr('cvel').reshape(-1, 6)
    forces = contact_world_forces(o, m)
    sb, sp, sq = m['site_bodyid'].astype(int), m['site_pos'].reshape(-1, 3), m['site_quat'].reshape(-1, 4)
    rows = np.zeros((len(names), W))
    for i, (name, kind) in enumerate(zip(names, kinds)):
        if kind == 0:
            b = list(m['names_body']).index(name)
            assert b < nb
            rows[i, POS:POS + 3], rows[i, QUAT:QUAT + 4], rows[i, VEL:VEL + 6] = xpos[b], xquat[b], cvel[b]
            for b1, b2, F in forces:
                if b1 == b:
                    rows[i, CFRC:CFRC + 3] -= F
                elif b2 == b:
                    rows[i, CFRC:CFRC + 3] += F
        else:
            s = list(m['names_site']).index(name)
            b = sb[s]
            rows[i, POS:POS + 3] = xpos[b] + xmat[b] @ sp[s]
            rows[i, QUAT:QUAT + 4] = mat2quat(quat2mat(mul_quat(xquat[b], sq[s])))
    return rows


def _compare(model, fp32, nticks=800, every=25, extra_pd=None):
    """stance for half the ticks, then a fall with the motors off; frames of every body and site checked every `every` ticks"""
    import oracle as O
    O.build(ref=False)
    m = omodel(model)
    names, kinds = all_frames(model)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    e = FrameSim(model, fp32=fp32)
    assert e.set_frames(names, kinds) == 0
    e.forward()
    stance, fall = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN), O.make_pd()
    worst = dict(pos=0.0, vel=0.0, cfrc=0.0)
    scale = dict(vel=0.0, cfrc=0.0)   # largest magnitude met, for the fp32 bars
    touched = set()
    for k in range(nticks):
        u, row = (stance, PD_ROW) if k < nticks // 2 else (fall, ZERO_ROW)
        o.step_pd(u)
        e.step(row)
        if k % every == every - 1:
            got, want = e.frames(), oracle_frames(o, m, names, kinds)
            worst['pos'] = max(worst['pos'], np.abs(got[:, :VEL] - want[:, :VEL]).max())
            worst['vel'] = max(worst['vel'], np.abs(got[:, VEL:CFRC] - want[:, VEL:CFRC]).max())
            worst['cfrc'] = max(worst['cfrc'], np.abs(got[:, CFRC:] - want[:, CFRC:]).max())
            scale['vel'] = max(scale['vel'], np.abs(want[:, VEL:CFRC]).max())
            scale['cfrc'] = max(scale['cfrc'], np.abs(want[:, CFRC:]).max())
            touched.update(i for i in range(len(names)) if np.abs(want[i, CFRC:]).max() > 0)
    return worst, scale, touched, names


@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_frames_follow_the_oracle_fp64(model):
    worst, _, touched, names = _compare(model, False)
    print(model, worst, sorted(names[i] for i in touched))
    assert worst['pos'] <= 1e-10 and worst['vel'] <= 1e-8 and worst['cfrc'] <= 1e-8, worst
    assert len(touched) >= 3   # both feet and, after the fall, more of the robot (or the cup) carry contact forces


@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_frames_follow_the_oracle_fp32(model):
    """fp32: poses within 1e-4; velocities and contact forces within 1e-3 of the largest magnitude met (the fall amplifies last-bit differences of
    the single-precision trajectory; the forces reach hundreds of newtons)"""
    worst, scale, _, _ = _compare(model, True)
    print(model, worst, scale)
    assert worst['pos'] <= 1e-4 and worst['vel'] <= 1e-3 * scale['vel'] and worst['cfrc'] <= 1e-3 * scale['cfrc'], (worst, scale)


def test_contact_decode_of_this_file_is_the_oracle_foot_forces():
    """the wrench restatement above agrees with the oracle's own cassie_sim_foot_forces (osim_foot_forces)"""
    import oracle as O
    O.build(ref=False)
    m = omodel('cassie')
    o = O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    names = ['left-foot', 'right-foot']
    for _ in range(300):
        o.step_pd(u)
    rows = oracle_frames(o, m, names, [0, 0])
    ff = o.foot_forces()
    assert np.abs(rows[0, CFRC:CFRC + 3] - ff[0:3]).max() < 1e-12 and np.abs(rows[1, CFRC:CFRC + 3] - ff[6:9]).max() < 1e-12
    assert np.abs(ff).max() > 1


@pytest.mark.parametrize('fp32', [False, True])
def test_foot_frames_equal_aux_bitwise(fp32):
    """the two foot bodies' velocity and force slots are bitwise aux's foot velocities and foot forces of the same launch"""
    e = FrameSim('cassie', fp32=fp32)
    assert e.set_frames(['left-foot', 'right-foot'], [0, 0]) == 0
    e.forward()
    for k in range(300):
        e.step(PD_ROW)
        fr, aux = e.frames(), e.get('aux')
        assert np.array_equal(fr[0, VEL:CFRC], aux[30:36]) and np.array_equal(fr[1, VEL:CFRC], aux[36:42]), k
        assert np.array_equal(fr[0, CFRC:CFRC + 6], aux[0:6]) and np.array_equal(fr[1, CFRC:CFRC + 6], aux[6:12]), k
    assert np.abs(aux[0:12]).max() > 1


@pytest.mark.parametrize('aux_on', [True, False])
def test_frames_change_nothing_else(aux_on):
    """a frame row leaves qpos, qvel, obs, aux and the counters bitwise as a run without one; with the aux row off too (the frames alone decode the
    contact list and copy cdof)"""
    a, b = FrameSim('cassie'), FrameSim('cassie')
    if not aux_on:
        a.plain_aux_off()
        b.plain_aux_off()
    names, kinds = all_frames('cassie')
    assert b.set_frames(names, kinds) == 0
    a.forward()
    b.forward()
    for k in range(600):
        row = PD_ROW if k < 300 else ZERO_ROW
        a.step(row)
        b.step(row)
        for f in ('qpos', 'qvel', 'obs', 'counters') + (('aux',) if aux_on else ()):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    assert np.abs(b.frames()[:, CFRC:]).max() > 0


def test_forward_fills_every_slot():
    """mode 1 (mj_forward, as at init and reset) fills poses, velocities and forces like a step"""
    import oracle as O
    O.build(ref=False)
    m = omodel('cassie')
    names, kinds = all_frames('cassie')
    e = FrameSim('cassie')
    assert e.set_frames(names, kinds) == 0
    e.forward()
    o = O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
    o.forward()
    got, want = e.frames(), oracle_frames(o, m, names, kinds)
    assert np.abs(got - want).max() < 1e-10
    assert np.abs(got[:, POS:POS + 3]).max() > 0.5


def test_set_frames_errors():
    e = FrameSim('cassie')
    assert e.set_frames(['no-such-body'], [0]) == -1
    assert e.set_frames(['left-toe'], [0]) == -1           # a site named as a body
    assert e.set_frames(['cassie-pelvis'], [2]) == -1      # unknown kind
    assert e.set_frames(['cassie-pelvis'] * 65, [0] * 65) == -1
    assert e.set_frames(['world', 'cassie-pelvis', 'left-toe'], [0, 0, 1]) == 0
    assert e.frames().shape == (3, W)


def oracle_jacobian(O, model, qpos, name, kind):
    """cassie_sim_get_jacobian_full(_site) restated on the oracle at `qpos`: kinematics and centre of mass of that state (a fresh oracle, forward),
    then mj_jac at xpos / site_xpos: jacp = cdof_lin + cdof_ang x (point - subtree_com[root]), jacr = cdof_ang over the dofs of the body's chain"""
    m = omodel(model)
    o = O.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    o.arr('qpos')[:] = qpos[:o.nq]
    o.forward()
    nv = o.nv
    cdof, com = o.arr('cdof').reshape(nv, 6), o.arr('subtree_com').reshape(-1, 3)
    xpos, xmat = o.arr('xpos').reshape(-1, 3), o.arr('xmat').reshape(-1, 3, 3)
    if kind == 0:
        b = list(m['names_body']).index(name)
        pt = xpos[b]
    else:
        s = list(m['names_site']).index(name)
        b = int(m['site_bodyid'][s])
        pt = xpos[b] + xmat[b] @ m['site_pos'].reshape(-1, 3)[s]
    parent, dofb, root = m['body_parentid'].astype(int), m['dof_bodyid'].astype(int), m['body_rootid'].astype(int)
    chain, a = set(), b
    while a > 0:
        chain.add(a)
        a = parent[a]
    jp, jr = np.zeros((3, nv)), np.zeros((3, nv))
    for i in range(nv):
        if dofb[i] in chain:
            jr[:, i] = cdof[i, :3]
            jp[:, i] = cdof[i, 3:] + np.cross(cdof[i, :3], pt - com[root[b]])
    o.close()
    return jp, jr


def emu_jacobian(e, f, nv):
    out = np.zeros(240)
    fr_lib().emu_fr_jacobian.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double)]
    assert fr_lib().emu_fr_jacobian(e.h, f, out.ctypes.data_as(C.POINTER(C.c_double))) == 0
    j = out.reshape(6, 40)
    assert not j[:, nv:].any()
    return j[:3, :nv], j[3:, :nv]


@pytest.mark.parametrize('model', ['cassie', 'cassie_hfield', 'cassie_tray_box'])
def test_jacobians_follow_the_oracle(oracle_mod, model):
    """mode 4 for every body and site at states of a stance and a fall, fp64 within 1e-10 (the tray box: 38 columns, the cup's own 6)"""
    names, kinds = all_frames(model)
    e = FrameSim(model)
    assert e.set_frames(names, kinds) == 0
    e.forward()
    nq = omodel(model)['qpos_spring'].size
    nv = 38 if model == 'cassie_tray_box' else 32
    worst = 0.0
    for k in range(400):
        e.step(PD_ROW if k < 200 else ZERO_ROW)
        if k % 100 == 99:
            q = e.get('qpos')[:nq]
            for f, (name, kind) in enumerate(zip(names, kinds)):
                jp, jr = emu_jacobian(e, f, nv)
                wp, wr = oracle_jacobian(oracle_mod, model, q, name, kind)
                worst = max(worst, np.abs(jp - wp).max(), np.abs(jr - wr).max())
    print(model, worst)
    assert worst <= 1e-10
    if model == 'cassie_tray_box':
        jp, jr = emu_jacobian(e, names.index(omodel(model)['names_body'][-1]), nv)
        assert np.abs(jp[:, 32:]).max() > 0.5 and not jp[:, :32].any()   # the cup moves with its own dofs only


@pytest.mark.parametrize('fp32', [False, True])
def test_jacobian_launch_leaves_the_state_alone(fp32):
    """mode 4 writes the Jacobian row only: the state, the rows and the next steps are bitwise those of a twin that never asked"""
    names, kinds = all_frames('cassie')
    a, b = FrameSim('cassie', fp32=fp32), FrameSim('cassie', fp32=fp32)
    for x in (a, b):
        assert x.set_frames(names, kinds) == 0
        x.forward()
    for k in range(300):
        a.step(PD_ROW)
        b.step(PD_ROW)
        if k % 30 == 0:
            emu_jacobian(b, k % len(names), 32)
            for f in ('qpos', 'qvel', 'obs', 'aux', 'counters', 'cst', 'qacc_ws'):
                assert np.array_equal(a.get(f), b.get(f)), (k, f)
            assert np.array_equal(a.frames(), b.frames())
