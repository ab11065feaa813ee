"""Register spills of the step-kernel instances with per-environment terrain (build.py TERRAIN_INSTANCES), as the assembler reports them for sm_90a (no
GPU needed), against their counterparts without it."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
TERRAIN_SPILL_LIMITS = {
    'f02f': (264, 400), 'f12f': (440, 904), 'f22f': (264, 416), 'd02f': (988, 1392), 'd12f': (1228, 2156), 'd22f': (992, 1408),
    'f13f': (352, 768), 'd13f': (1148, 2108),
}
COUNTERPART = {'f02f': 'f0f', 'f12f': 'f1f', 'f22f': 'f2f', 'd02f': 'd0f', 'd12f': 'd1f', 'd22f': 'd2f', 'f13f': 'f11f', 'd13f': 'd11f'}
# instances more than this many spill bytes (stores or loads) above their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 64


def test_every_terrain_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.TERRAIN_INSTANCES) == sorted(TERRAIN_SPILL_LIMITS)
    assert all(feat & 32 for *_, feat in mod.TERRAIN_INSTANCES)
    assert not any(feat & 32 for *_, feat in mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES)
    others = {t: (real, dr, feat) for t, real, dr, feat in mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES}
    for t, real, dr, feat in mod.TERRAIN_INSTANCES:   # each has a counterpart without terrain rows of the same precision, kind and features
        assert others[COUNTERPART[t]] == (real, dr, feat & ~32)


@pytest.mark.parametrize('tag', sorted(TERRAIN_SPILL_LIMITS))
def test_terrain_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without terrain rows %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = TERRAIN_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(TERRAIN_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
