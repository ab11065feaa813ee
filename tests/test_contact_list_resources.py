"""Register spills of the step-kernel instances with contact lists (build.py CONTACT_LIST_INSTANCES), as the assembler reports them for sm_90a (no
GPU needed), against the F_FR chain twins they are the F_CL twins of."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

F_FR, F_XF, F_TC, F_CL = 16, 1024, 2048, 4096
# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
CONTACT_LIST_SPILL_LIMITS = {
    'f117d7': (400, 888), 'd117d7': (1176, 2160), 'f117df': (432, 1072), 'd117df': (1184, 2260), 'f117ff': (432, 1072), 'd117ff': (1184, 2260),
}
COUNTERPART = {'f117d7': 'f17d7', 'd117d7': 'd17d7', 'f117df': 'f17df', 'd117df': 'd17df', 'f117ff': 'f17ff', 'd117ff': 'd17ff'}
# instances that spill more bytes (stores or loads) than their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 0


def test_every_contact_list_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.CONTACT_LIST_INSTANCES) == sorted(CONTACT_LIST_SPILL_LIMITS)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES + mod.ACTUATOR_INSTANCES + \
        mod.MECHANICS_INSTANCES + mod.CONTACT_INSTANCES + mod.APPLIED_INSTANCES + mod.TRACE_INSTANCES
    assert not any(feat & F_CL for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.CONTACT_LIST_INSTANCES:   # each is its F_FR chain twin of the same precision, kind and features, plus F_CL and nothing else
        assert feat & F_CL and others[COUNTERPART[t]] == (real, dr, feat & ~F_CL)
        assert dr == 1 and feat & F_XF and feat & F_FR and not feat & F_TC and COUNTERPART[t] in [x for x, *_ in mod.APPLIED_INSTANCES]


@pytest.mark.parametrize('tag', sorted(CONTACT_LIST_SPILL_LIMITS))
def test_contact_list_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without lists %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = CONTACT_LIST_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(CONTACT_LIST_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
