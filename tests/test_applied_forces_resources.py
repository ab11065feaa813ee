"""Register spills of the step-kernel instances with per-environment applied forces (build.py APPLIED_INSTANCES), as the assembler reports them for
sm_90a (no GPU needed), against their counterparts without them: f04 / f24 for the plain twins, the F_CT instances for the chain twins."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

F_BOX, F_CT, F_XF = 4, 512, 1024
# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
APPLIED_SPILL_LIMITS = {
    'f0404': (96, 112), 'f2404': (112, 136),
    'f17c4': (260, 504), 'f17d7': (388, 864), 'd17d7': (1164, 2072), 'f17df': (420, 1036), 'd17df': (1184, 2216), 'f17ff': (420, 1036), 'd17ff': (1184, 2216),
}
COUNTERPART = {'f0404': 'f04', 'f2404': 'f24', 'f17c4': 'f13c4', 'f17d7': 'f13d7', 'd17d7': 'd13d7', 'f17df': 'f13df', 'd17df': 'd13df', 'f17ff': 'f13ff',
               'd17ff': 'd13ff'}
# instances that spill more bytes (stores or loads) than their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 0


def test_every_applied_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.APPLIED_INSTANCES) == sorted(APPLIED_SPILL_LIMITS)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES + mod.ACTUATOR_INSTANCES + \
        mod.MECHANICS_INSTANCES + mod.CONTACT_INSTANCES
    assert not any(feat & F_XF for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.APPLIED_INSTANCES:   # each is its counterpart of the same precision, kind and features, plus F_XF
        assert feat & F_XF and others[COUNTERPART[t]] == (real, dr, feat & ~F_XF)
        assert (dr == 1 and feat & F_CT) or (dr != 1 and feat == F_BOX | F_XF and real == 'float')   # chain twins extended, plain twins the push workload's


@pytest.mark.parametrize('tag', sorted(APPLIED_SPILL_LIMITS))
def test_applied_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without applied rows %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = APPLIED_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(APPLIED_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
