"""Per-environment contact softness on the fp64 oracle, for tests/test_env_contact.py and tests/test_gpu_env_contact.py.

The oracle gets solref / solimp / solmix per geom through a temporary copy of its model table (mechanics_support.oracle_with): the geom_solref, geom_solimp
and geom_solmix lines, which its collision stage mixes per contact as mj_contactParam does."""
import numpy as np

from mechanics_support import oracle_with, table


def model_contact(model):
    """(solref [ngeom, 2], solimp [ngeom, 5], solmix [ngeom]): the model's values, as the batch's get reports them without rows"""
    t = table(model)
    return t['geom_solref'].reshape(-1, 2).copy(), t['geom_solimp'].reshape(-1, 5).copy(), t['geom_solmix'].copy()


def colliding(model):
    """geoms that can make contact (contype or conaffinity non-zero)"""
    t = table(model)
    return [g for g in range(len(t['geom_contype'])) if t['geom_contype'][g] or t['geom_conaffinity'][g]]


def random_contact(model, seed, base=None):
    """seeded values of the kinds users randomise, per colliding geom: timeconst x [0.6, 3], dampratio x [0.5, 1.5], dmin and dmax +-0.04 (dmin <= dmax
    kept), width x [0.5, 4], midpoint in [0.3, 0.7], power in [1, 3], solmix in [0.2, 2].  Every geom draws its own values, so the two feet differ and the
    floor differs from the stairs.  base: the values to start from (solref, solimp, solmix), by default the oracle table's"""
    sr, si, sm = [np.array(v, float) for v in (model_contact(model) if base is None else base)]
    rng = np.random.default_rng(seed)
    for g in colliding(model):
        sr[g, 0] *= rng.uniform(0.6, 3.0)
        sr[g, 1] *= rng.uniform(0.5, 1.5)
        dmax = np.clip(si[g, 1] + rng.uniform(-0.04, 0.04), 0.5, 0.99)
        si[g, 0] = np.clip(si[g, 0] + rng.uniform(-0.04, 0.04), 0.5, dmax)
        si[g, 1] = dmax
        si[g, 2] *= rng.uniform(0.5, 4.0)
        si[g, 3] = rng.uniform(0.3, 0.7)
        si[g, 4] = rng.uniform(1.0, 3.0)
        sm[g] = rng.uniform(0.2, 2.0)
    return sr, si, sm


def contact_oracle(O, model, solref=None, solimp=None, solmix=None, **lines):
    """an fp64 oracle of `model` whose geom_solref [ngeom, 2], geom_solimp [ngeom, 5] and geom_solmix [ngeom] are the given ones (None: the table's);
    lines: further table arrays by name (geom_friction, body_inertia, ...), each given whole"""
    return oracle_with(O, model, geom_solref=solref, geom_solimp=solimp, geom_solmix=solmix, **lines)
