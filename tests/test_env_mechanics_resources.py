"""Register spills of the step-kernel instances with per-environment mechanics (build.py MECHANICS_INSTANCES), as the assembler reports them for sm_90a
(no GPU needed), against their counterparts without them: the F_AC instances they are the F_MC twins of."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

F_AC, F_MC = 128, 256
# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
MECHANICS_SPILL_LIMITS = {
    'f11c4': (268, 520), 'f11d7': (392, 852), 'd11d7': (1164, 2048), 'f11df': (384, 824), 'd11df': (1184, 2180), 'f11ff': (384, 824), 'd11ff': (1184, 2180),
}
COUNTERPART = {'f11c4': 'f1c4', 'f11d7': 'f1d7', 'd11d7': 'd1d7', 'f11df': 'f1df', 'd11df': 'd1df', 'f11ff': 'f1ff', 'd11ff': 'd1ff'}
# instances that spill more bytes (stores or loads) than their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 0


def test_every_mechanics_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.MECHANICS_INSTANCES) == sorted(MECHANICS_SPILL_LIMITS)
    assert all(feat & F_MC and feat & F_AC and dr == 1 for _, _, dr, feat in mod.MECHANICS_INSTANCES)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES + mod.ACTUATOR_INSTANCES
    assert not any(feat & F_MC for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.MECHANICS_INSTANCES:   # each is the F_AC twin's of the same precision, kind and features, plus F_MC
        assert others[COUNTERPART[t]] == (real, dr, feat & ~F_MC)


@pytest.mark.parametrize('tag', sorted(MECHANICS_SPILL_LIMITS))
def test_mechanics_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without mechanics rows %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = MECHANICS_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(MECHANICS_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
