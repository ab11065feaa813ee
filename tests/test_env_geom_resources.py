"""Register spills of the step-kernel instances that read the static geoms' placement from per-environment rows (build.py ENV_GEOM_INSTANCES), as the
assembler reports them for sm_90a (no GPU needed; the shipped instances are checked by tests/test_step_resources.py)."""
import importlib.util
import os

import pytest

from conftest import REPO
from test_step_resources import SPILL_LIMITS, kernel_resources

# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a.  The F_BOX | F_EG instances stay within their
# shared-placement counterparts' limits; the F_ALL | F_EG ones exceed theirs by 8-32 bytes (DESIGN.md section 5).  Lower them when an edit lowers the spills.
ENV_GEOM_SPILL_LIMITS = {
    'f0c': (32, 40), 'f1c': (188, 292), 'f2c': (44, 60),
    'f0f': (256, 400), 'f1f': (444, 940), 'f2f': (264, 416),
    'd0f': (972, 1392), 'd1f': (1220, 2152), 'd2f': (984, 1408),
}
COUNTERPART = {'f0c': 'f04', 'f1c': 'f14', 'f2c': 'f24', 'f0f': 'f07', 'f1f': 'f17', 'f2f': 'f27', 'd0f': 'd07', 'd1f': 'd17', 'd2f': 'd27'}


def _build_module():
    spec = importlib.util.spec_from_file_location('_cassie_b200_build', os.path.join(REPO, 'cassie-mujoco-sim_b200', 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_every_env_geom_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.ENV_GEOM_INSTANCES) == sorted(ENV_GEOM_SPILL_LIMITS)
    assert all(feat & 8 for *_, feat in mod.ENV_GEOM_INSTANCES) and not any(feat & 8 for *_, feat in mod.INSTANCES)
    shipped = {t: (real, dr, feat) for t, real, dr, feat in mod.INSTANCES}
    for t, real, dr, feat in mod.ENV_GEOM_INSTANCES:   # each has a shared-placement counterpart of the same precision and kind
        assert shipped[COUNTERPART[t]] == (real, dr, feat & ~8)


@pytest.mark.parametrize('tag', sorted(ENV_GEOM_SPILL_LIMITS))
def test_env_geom_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    base = SPILL_LIMITS[COUNTERPART[tag]]
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (shared placement %s: limit %d / %d)' % (tag, stack, st, ld, COUNTERPART[tag], *base))
    max_st, max_ld = ENV_GEOM_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))
