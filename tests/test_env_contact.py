"""Per-environment contact softness (cassie_batch_set_env_contact): the product's stepper source in the host emulation, with each contact row's solref and
solimp mixed from the environment's per-geom solref / solimp / solmix (the F_CT instances) instead of the pair's parameter record.  The GPU twins are in
tests/test_gpu_env_contact.py.

The emulation is tests/emu/emu_env_contact.cpp, built into its own library here.  The fp64 oracle gets the same values through a temporary copy of its
model table (tests/contact_support.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
from contact_support import colliding, contact_oracle, model_contact, random_contact
from mechanics_support import table

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
CT_SLOT, CT_SOLREF, CT_SOLIMP, CT_SOLMIX, CONTACT_W = 8, 0, 2, 7, 256   # devmodel.h CT_*
D_EFC_R, D_EFC_AREF = 1380, 1444   # devmodel.h D_*

_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_env_contact.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_env_contact.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci = C.c_void_p, C.POINTER(C.c_double), C.c_int
        L.emu_ct_new.restype = vp
        L.emu_ct_new.argtypes = [C.c_char_p, ci]
        for n in ('emu_ct_free', 'emu_ct_forward', 'emu_ct_ngeom'):
            getattr(L, n).argtypes = [vp]
        L.emu_ct_mode.argtypes = [vp, ci]
        L.emu_ct_set.argtypes = [vp, dp, dp, dp]
        L.emu_ct_poke.argtypes = [vp, ci, C.c_double]
        L.emu_ct_row.argtypes = [vp, dp]
        L.emu_ct_model.argtypes = [vp, dp, dp, dp, C.POINTER(C.c_int)]
        L.emu_ct_step.argtypes = [vp, dp, ci]
        L.emu_ct_check.argtypes = [vp, ci, vp, vp, vp, vp, C.c_char_p]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return None if a is None else np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


class CtSim:
    """one emulated environment; mode 0 runs the extended F_ALL source, 1 the F_MC source with model-valued rows, 2 the F_MC | F_CT source"""

    def __init__(self, model, fp32=False, mode=2):
        self.L = lib()
        self.h = self.L.emu_ct_new(os.path.join(MODELS, model + '.cmodel').encode(), 1 if fp32 else 0)
        assert self.h
        self.L.emu_ct_mode(self.h, mode)
        self.name = model

    def close(self):
        if self.h:
            self.L.emu_ct_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def put(self, name, arr):
        a = np.ascontiguousarray(arr, dtype=np.float64)
        assert self.L.emu_set(self.h, name.encode(), _dp(a), len(a)) >= 0, name

    def set_contact(self, solref=None, solimp=None, solmix=None):
        self._keep = [None if a is None else np.ascontiguousarray(a, dtype=np.float64).ravel() for a in (solref, solimp, solmix)]
        self.L.emu_ct_set(self.h, *[_dp(a) for a in self._keep])

    def model(self):
        """(solref [ngeom, 2], solimp [ngeom, 5], solmix [ngeom]) of the product's compiled model, and each geom's device slot (-1: none)"""
        ng = self.L.emu_ct_ngeom(self.h)
        out = [np.zeros((ng, 2)), np.zeros((ng, 5)), np.zeros(ng)]
        slot = np.zeros(ng, dtype=np.int32)
        self.L.emu_ct_model(self.h, *[_dp(v) for v in out], slot.ctypes.data_as(C.POINTER(C.c_int)))
        return out, slot

    def row(self):
        out = np.zeros(CONTACT_W)
        self.L.emu_ct_row(self.h, out.ctypes.data_as(C.POINTER(C.c_double)))
        return out

    def step(self, pd50=PD_ROW, nticks=1):
        self.L.emu_ct_step(self.h, _dp(pd50), nticks)

    def forward(self):
        self.L.emu_ct_forward(self.h)


def _body_geom(model, body):
    t = table(model)
    b = t['names_body'].index(body)
    return [g for g in colliding(model) if t['geom_bodyid'][g] == b][0]


# ------------------------------------------------------------------ 1. rows at the model's values are the F_MC source, bitwise
@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box', 'cassie_hfield', 'cassie_depth'])
@pytest.mark.parametrize('fp32', [False, True])
def test_model_rows_are_bitwise_the_mechanics_source(model, fp32):
    """every shipped model gives its colliding geoms equal values or resolves the pair by priority, so the mixed values are the record's exactly"""
    a, b = CtSim(model, fp32, mode=1), CtSim(model, fp32, mode=2)
    b.set_contact(*b.model()[0])   # what the setter stores for the model's values
    for k in range(300):
        a.step()
        b.step()
        for f in ('qpos', 'qvel', 'obs', 'aux', 'cst', 'counters'):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    a.close()
    b.close()


# ------------------------------------------------------------------ 2. against the oracle
@pytest.mark.parametrize('model', ['cassie', 'cassie_mass', 'cassie_tray_box', 'cassie_hfield'])
def test_env_contact_follows_the_oracle(oracle_mod, model):
    """fp64: qpos within 1e-9 of the oracle with the same geom_solref / solimp / solmix over 500 ticks, the same PGS iteration count every tick;
    cassie_tray_box's cup contacts bring ticks with more than 32 constraint rows (the non-dense solve) into the run"""
    sr, si, sm = random_contact(model, 21)
    for left, right in (('left-foot', 'right-foot'),):
        gl, gr = _body_geom(model, left), _body_geom(model, right)
        assert not np.array_equal(sr[gl], sr[gr]) and not np.array_equal(si[gl], si[gr])
    o = contact_oracle(oracle_mod, model, sr, si, sm)
    o.set_caps()
    e = CtSim(model)
    e.set_contact(sr, si, sm)
    e.forward()
    o.forward()
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    worst, iters_equal, big = 0.0, True, 0
    for k in range(500):
        o.step_pd(u)
        e.step()
        worst = max(worst, np.abs(e.get('qpos')[:o.nq] - o.arr('qpos')).max())
        c = e.get('counters')
        iters_equal = iters_equal and int(c[3]) == o.get_int('solver_iter')
        big += int(c[0]) > 32
    print(model, 'qpos %.2e, %d ticks with nefc > 32' % (worst, big))
    assert worst < 1e-9 and iters_equal, (model, worst, iters_equal)
    assert big > 0 or model != 'cassie_tray_box', model
    # the values change the motion: the model's own trajectory is elsewhere
    o0 = contact_oracle(oracle_mod, model)
    o0.set_caps()
    o0.forward()
    for k in range(500):
        o0.step_pd(u)
    assert np.abs(o0.arr('qpos') - o.arr('qpos')).max() > 1e-5
    e.close()
    o.close()
    o0.close()


def test_row_constants_follow_the_oracle(oracle_mod):
    """at a contact state: the R and aref of every constraint row (the debug dump) against the oracle's efc_R and efc_aref, within 1e-10 relative"""
    model = 'cassie'
    sr, si, sm = random_contact(model, 7)
    o = contact_oracle(oracle_mod, model, sr, si, sm)
    e = CtSim(model)
    e.set_contact(sr, si, sm)
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for _ in range(120):
        o.step_pd(u)
        e.step()
    n = o.get_int('nefc')
    assert n == int(e.get('counters')[0]) and o.get_int('ncon') > 0
    dbg = e.get('dbg')
    for key, name in ((D_EFC_R, 'efc_R'), (D_EFC_AREF, 'efc_aref')):
        want = o.arr(name)[:n]
        assert np.abs(dbg[key:key + n] - want).max() <= 1e-10 * np.abs(want).max(), name
    e.close()
    o.close()


# ------------------------------------------------------------------ 3. the mixing rules
def _run(model, rows, ticks=300, fp32=False):
    e = CtSim(model, fp32)
    e.set_contact(*rows)
    out = []
    for _ in range(ticks):
        e.step()
        out.append(e.get('qpos'))
    e.close()
    return np.array(out)


def test_priority_takes_the_floor(oracle_mod):
    """cassie_mass's floor has priority 1: a foot's values leave the floor contacts bitwise unchanged; the floor's change them"""
    model = 'cassie_mass'
    base = model_contact(model)
    ref = _run(model, base)
    foot = [np.array(v) for v in base]
    g = _body_geom(model, 'left-foot')
    foot[0][g] = [0.03, 0.3]
    foot[1][g] = [0.5, 0.6, 0.01, 0.4, 1.5]
    foot[2][g] = 5.0
    assert np.array_equal(_run(model, foot), ref)
    floor = [np.array(v) for v in base]
    floor[0][0] = [0.02, 0.7]
    assert np.abs(_run(model, floor) - ref).max() > 1e-6


def test_solmix_weights():
    """solmix 0 on one geom takes the other geom's values; solmix 0 on both mixes half and half"""
    model = 'cassie'
    gl, gr = _body_geom(model, 'left-foot'), _body_geom(model, 'right-foot')
    base = model_contact(model)
    x = [np.array(v) for v in base]
    for g in (gl, gr):   # x: the feet soft, and their solmix 0: the floor's values apply
        x[0][g] = [0.03, 0.4]
        x[1][g] = [0.6, 0.7, 0.01, 0.3, 1.2]
        x[2][g] = 0.0
    ref = _run(model, base)
    assert np.array_equal(_run(model, x), ref)
    half = [np.array(v) for v in x]   # the floor's solmix 0 as well: both below the threshold, mix 0.5, as with solmix 1 on both
    half[2][0] = 1.0
    for g in (gl, gr):
        half[2][g] = 1.0
    y = [np.array(v) for v in x]
    y[2][0] = 0.0
    got, want = _run(model, y), _run(model, half)
    assert np.array_equal(got, want) and np.abs(got - ref).max() > 1e-6


def test_standard_against_direct_takes_the_min(oracle_mod):
    """a direct-form foot (stiffness, damping negated) against the standard-form floor: the elementwise min, which is the foot's pair -- the same motion as
    both feet and the floor in that direct form, and the oracle's"""
    model = 'cassie'
    gl, gr = _body_geom(model, 'left-foot'), _body_geom(model, 'right-foot')
    base = model_contact(model)
    d = [np.array(v) for v in base]
    for g in (gl, gr):
        d[0][g] = [-40000.0, -400.0]
    both = [np.array(v) for v in d]
    both[0][0] = [-40000.0, -400.0]
    got = _run(model, d)
    assert np.array_equal(got, _run(model, both))
    o = contact_oracle(oracle_mod, model, *d)
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for _ in range(300):
        o.step_pd(u)
    assert np.abs(got[-1][:o.nq] - o.arr('qpos')).max() < 1e-9
    o.close()


def test_timeconst_below_two_steps_is_floored():
    """a timeconst below 2 h (h = 0.5 ms) acts as 2 h, bit for bit"""
    model = 'cassie'
    a, b = [np.array(v) for v in model_contact(model)], [np.array(v) for v in model_contact(model)]
    for g in colliding(model):
        a[0][g, 0] = 1e-4
        b[0][g, 0] = 2 * 0.0005
    got = _run(model, a)
    assert np.array_equal(got, _run(model, b)) and np.abs(got - _run(model, model_contact(model))).max() > 1e-7


# ------------------------------------------------------------------ 4. rows, slots and the setter's check
def test_row_layout_and_unslotted_geoms():
    """slot k holds device geom k's solref, solimp and solmix; slots without a geom stay zero; entries of geoms without a collision slot are ignored"""
    model = 'cassie'
    sr, si, sm = random_contact(model, 4)
    e = CtSim(model)
    (msr, msi, msm), slot = e.model()
    visual = [g for g in range(len(slot)) if slot[g] < 0]
    assert visual and sorted(g for g in range(len(slot)) if slot[g] >= 0) == colliding(model)
    for g in visual:   # any value for a visual geom, even one the check would refuse for a colliding geom
        sr[g], si[g], sm[g] = [np.nan, 1.0], [2.0] * 5, -1.0
    e.set_contact(sr, si, sm)
    r = e.row()
    used = set()
    for g in colliding(model):
        s = slot[g]
        used.add(s)
        q = r[CT_SLOT * s:CT_SLOT * (s + 1)]
        assert np.array_equal(q[CT_SOLREF:CT_SOLREF + 2], sr[g]) and np.array_equal(q[CT_SOLIMP:CT_SOLIMP + 5], si[g]) and q[CT_SOLMIX] == sm[g], g
    assert not any(r[CT_SLOT * s:CT_SLOT * (s + 1)].any() for s in range(32) if s not in used)
    assert np.isfinite(r).all()
    n = 2
    assert _check(e, n, [np.tile(v, (n, 1, 1))[:, :, :] if v.ndim == 2 else np.tile(v, (n, 1)) for v in (sr, si, sm)])[0] == 0
    # the run with the visual entries is the run without them, bit for bit
    f = CtSim(model)
    f.set_contact(*random_contact(model, 4))
    for _ in range(100):
        e.step()
        f.step()
    assert np.array_equal(e.get('qpos'), f.get('qpos'))
    e.close()
    f.close()


def _check(s, n, parts, mask=None):
    why = C.create_string_buffer(512)
    arr = [None if a is None else np.ascontiguousarray(a, dtype=np.float64) for a in parts]
    m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
    r = s.L.emu_ct_check(s.h, n, *[None if a is None else a.ctypes.data_as(C.c_void_p) for a in arr], None if m is None else m.ctypes.data_as(C.c_void_p), why)
    return r, why.value.decode()


@pytest.mark.parametrize('model', ['cassie', 'cassie_tray_box'])
def test_setter_refusals(model):
    """the batch setter's check: every masked value before anything changes, with the environment, the geom and the field named; unmasked environments
    are not checked"""
    n = 3
    s = CtSim(model)
    (sr, si, sm), _ = s.model()
    base = [np.tile(sr, (n, 1, 1)), np.tile(si, (n, 1, 1)), np.tile(sm, (n, 1))]
    assert _check(s, n, base)[0] == 0
    assert _check(s, n, [None] * 3)[0] == 0
    ok = [v.copy() for v in base]
    g = colliding(model)[3]
    gname = table(model)['names_geom'][g]
    gname = str(g) if gname in ('', '-') else gname   # unnamed geoms are named by index
    ok[0][1, g] = [-1e4, -50.0]   # direct form
    ok[0][2, g] = [0.0, 0.0]      # direct form, no stiffness or damping
    ok[1][0, g] = [0.01, 0.99, 0.0, 0.5, 1.0]
    ok[2][2, g] = 0.0
    assert _check(s, n, ok)[0] == 0, _check(s, n, ok)[1]

    def bad(part, env, idx, value, words):
        p = [v.copy() for v in base]
        p[part][(env,) + idx] = value
        r, why = _check(s, n, p)
        assert r == 1 and all(w in why for w in words) and 'environment %d, geom %s:' % (env, gname) in why, (part, idx, value, why)
        m = [1] * n
        m[env] = 0
        assert _check(s, n, p, mask=m)[0] == 0   # a refused value in an unselected environment is not looked at

    bad(0, 1, (g, 0), np.nan, ['geom_solref', 'not finite'])
    bad(0, 2, (g, 1), np.inf, ['geom_solref', 'not finite'])
    bad(0, 0, (g,), [0.02, -1.0], ['geom_solref', 'mixed'])
    bad(0, 0, (g,), [-100.0, 1.0], ['geom_solref', 'mixed'])
    bad(0, 1, (g,), [0.0, 1.0], ['geom_solref', 'standard'])
    for k, name, v in ((0, 'dmin', 0.0), (0, 'dmin', 1.0), (1, 'dmax', 0.0), (1, 'dmax', 1.2), (3, 'midpoint', 0.0), (3, 'midpoint', 1.0)):
        bad(1, 1, (g, k), v, ['geom_solimp[%d]' % k, name, '(0, 1)'])
    bad(1, 2, (g, 2), -1e-3, ['geom_solimp[2]', 'width', '>= 0'])
    bad(1, 0, (g, 4), 0.5, ['geom_solimp[4]', 'power', '>= 1'])
    bad(1, 0, (g, 4), np.nan, ['geom_solimp[4]', 'not finite'])
    bad(2, 1, (g,), -0.1, ['geom_solmix', '>= 0'])
    bad(2, 2, (g,), np.inf, ['geom_solmix', 'not finite'])
    s.close()


# ------------------------------------------------------------------ 5. physics: softer ground sinks
def test_softer_ground_stands_lower():
    """a timeconst of 0.02 s instead of the model's 0.005 s: the robot stands measurably lower after 600 ticks"""
    model = 'cassie'
    base = model_contact(model)
    soft = [np.array(v) for v in base]
    for g in colliding(model):
        soft[0][g, 0] = 0.02
    z = {}
    for name, rows in (('model', base), ('soft', soft)):
        e = CtSim(model)
        e.set_contact(*rows)
        e.step(nticks=600)
        z[name] = e.get('qpos')[2]
        e.close()
    print('pelvis z after 600 ticks: model %.5f, timeconst 0.02 %.5f' % (z['model'], z['soft']))
    assert z['soft'] < z['model'] - 1e-3
