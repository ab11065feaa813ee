"""Per-environment mechanics on the fp64 oracle, for tests/test_env_mechanics.py and tests/test_gpu_env_mechanics.py.

The oracle gets link inertias, armatures and hinge springs through a temporary copy of its model table: the body_inertia, dof_armature, jnt_stiffness and
qpos_spring lines (MuJoCo's arrays; nothing else in the table changes, as when the reference writes them into the mjModel).  Its mj_setConst constants
stay the table's until just_set_const(), as in MuJoCo."""
import os
import tempfile

import numpy as np

from conftest import GOLDEN

HINGE = 3   # MuJoCo's mjJNT_HINGE


def table(model):
    """dict of the oracle's model table arrays the mechanics touch (floats or ints), plus names_body / names_jnt"""
    t = {ln.split()[0]: ln.split() for ln in open(os.path.join(GOLDEN, model + '.omodel')).read().split('\n') if ln.strip()}
    out = {}
    for k, v in t.items():
        if len(v) >= 3 and v[1] in ('F', 'I'):
            out[k] = np.array([float(x) for x in v[3:]]) if v[1] == 'F' else np.array([int(x) for x in v[3:]])
        else:
            out[k] = v[3:]
    return out


def model_values(model):
    """(inertia [nbody, 3], armature [nv], stiffness [njnt], springref [njnt]): the model's values, as the batch's get reports them without rows"""
    t = table(model)
    return t['body_inertia'].reshape(-1, 3).copy(), t['dof_armature'].copy(), t['jnt_stiffness'].copy(), t['qpos_spring'][t['jnt_qposadr']].copy()


def changeable_bodies(model):
    """bodies whose inertia the verb may change: not the world, not welded to the world, not the extra free body (cassie_tray_box's last body)"""
    t = table(model)
    nb = len(t['body_weldid'])
    xb = nb - 1 if model == 'cassie_tray_box' else -1
    return [b for b in range(1, nb) if t['body_weldid'][b] != 0 and b != xb]


def random_mechanics(model, seed, base=None):
    """seeded values of the kinds users randomise: each changeable body's moments x [0.8, 1.2] (one factor per body, so A + B >= C holds), every main-tree
    armature x [0.5, 1.5], every sprung hinge's stiffness x [0.7, 1.3] and rest angle +-0.02 rad; base: the values to start from (inertia, armature,
    stiffness, springref), by default the oracle table's"""
    t = table(model)
    I, arm, k, q = [np.array(v, float) for v in (model_values(model) if base is None else base)]
    rng = np.random.default_rng(seed)
    for b in changeable_bodies(model):
        I[b] *= rng.uniform(0.8, 1.2)
    nvm = 32
    arm[:nvm] *= rng.uniform(0.5, 1.5, nvm)
    for j in range(len(k)):
        if t['jnt_type'][j] == HINGE and k[j] != 0:
            k[j] *= rng.uniform(0.7, 1.3)
            q[j] += rng.uniform(-0.02, 0.02)
    return I, arm, k, q


def oracle_with(O, model, inertia=None, armature=None, stiffness=None, springref=None, **lines):
    """an fp64 oracle of `model` whose body_inertia [nbody, 3], dof_armature [nv], jnt_stiffness [njnt] and the qpos_spring of each joint [njnt] (at its
    qposadr; only hinges' entries are written) are the given ones (None: the table's); lines: further table arrays by name (body_mass, body_pos,
    actuator_ctrlrange, ...), each given whole"""
    t = table(model)
    qs = t['qpos_spring'].copy()
    if springref is not None:
        for j, a in enumerate(t['jnt_qposadr']):
            if t['jnt_type'][j] == HINGE:
                qs[a] = springref[j]
    new = dict(body_inertia=inertia, dof_armature=armature, jnt_stiffness=stiffness, qpos_spring=None if springref is None else qs, **lines)
    lines = open(os.path.join(GOLDEN, model + '.omodel')).read().split('\n')
    for i, ln in enumerate(lines):
        w = ln.split()
        if w and w[0] in new and new[w[0]] is not None:
            lines[i] = ' '.join(w[:3] + [repr(float(x)) for x in np.asarray(new[w[0]], float).ravel()])
    with tempfile.TemporaryDirectory() as d:
        p = os.path.join(d, model + '.omodel')
        with open(p, 'w') as f:
            f.write('\n'.join(lines))
        return O.OracleSim(p)
