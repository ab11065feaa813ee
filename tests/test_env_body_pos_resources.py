"""Register spills of the step-kernel instances with per-environment body offsets (build.py BODY_POS_INSTANCES), as the assembler reports them for sm_90a
(no GPU needed), against their counterparts without them."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
BODY_POS_SPILL_LIMITS = {
    'f144': (244, 456), 'f157': (416, 844), 'd157': (1140, 2016), 'f15f': (360, 772), 'd15f': (1160, 2128), 'f17f': (360, 772), 'd17f': (1160, 2128),
}
COUNTERPART = {'f144': 'f14', 'f157': 'f117', 'd157': 'd117', 'f15f': 'f11f', 'd15f': 'd11f', 'f17f': 'f13f', 'd17f': 'd13f'}
# instances that spill more bytes (stores or loads) than their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 0


def test_every_body_pos_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.BODY_POS_INSTANCES) == sorted(BODY_POS_SPILL_LIMITS)
    assert all(feat & 64 and dr == 1 for _, _, dr, feat in mod.BODY_POS_INSTANCES)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES
    assert not any(feat & 64 for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.BODY_POS_INSTANCES:   # each has a counterpart without the rows of the same precision, kind and features
        assert others[COUNTERPART[t]] == (real, dr, feat & ~64)


@pytest.mark.parametrize('tag', sorted(BODY_POS_SPILL_LIMITS))
def test_body_pos_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without body-offset rows %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = BODY_POS_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(BODY_POS_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
