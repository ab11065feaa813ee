"""Register spills of the step-kernel instances with per-environment contact softness (build.py CONTACT_INSTANCES), as the assembler reports them for
sm_90a (no GPU needed), against their counterparts without them: the F_MC instances they are the F_CT twins of."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

F_MC, F_CT = 256, 512
# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
CONTACT_SPILL_LIMITS = {
    'f13c4': (260, 504), 'f13d7': (392, 852), 'd13d7': (1172, 2060), 'f13df': (424, 1012), 'd13df': (1192, 2196), 'f13ff': (424, 1012), 'd13ff': (1192, 2196),
}
COUNTERPART = {'f13c4': 'f11c4', 'f13d7': 'f11d7', 'd13d7': 'd11d7', 'f13df': 'f11df', 'd13df': 'd11df', 'f13ff': 'f11ff', 'd13ff': 'd11ff'}
# instances that spill more bytes (stores or loads) than their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 0


def test_every_contact_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.CONTACT_INSTANCES) == sorted(CONTACT_SPILL_LIMITS)
    assert all(feat & F_CT and feat & F_MC and dr == 1 for _, _, dr, feat in mod.CONTACT_INSTANCES)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES + mod.ACTUATOR_INSTANCES + \
        mod.MECHANICS_INSTANCES
    assert not any(feat & F_CT for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.CONTACT_INSTANCES:   # each is the F_MC twin's of the same precision, kind and features, plus F_CT
        assert others[COUNTERPART[t]] == (real, dr, feat & ~F_CT)


@pytest.mark.parametrize('tag', sorted(CONTACT_SPILL_LIMITS))
def test_contact_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without contact rows %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = CONTACT_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(CONTACT_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
