"""Register spills of the step-kernel instances with a per-tick trace (build.py TRACE_INSTANCES), as the assembler reports them for sm_90a (no GPU
needed), against the applied-force chain twins they are the F_TC twins of."""
import os

import pytest

from conftest import REPO
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

F_XF, F_TC = 1024, 2048
# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
TRACE_SPILL_LIMITS = {
    'f1fc4': (272, 536), 'f1fd7': (416, 1052), 'd1fd7': (1204, 2180), 'f1fdf': (444, 1160), 'd1fdf': (1212, 2276), 'f1fff': (444, 1160), 'd1fff': (1212, 2276),
}
COUNTERPART = {'f1fc4': 'f17c4', 'f1fd7': 'f17d7', 'd1fd7': 'd17d7', 'f1fdf': 'f17df', 'd1fdf': 'd17df', 'f1fff': 'f17ff', 'd1fff': 'd17ff'}
# instances that spill more bytes (stores or loads) than their counterpart must be explained in DESIGN.md section 5
EXPLAIN_ABOVE = 0


def test_every_trace_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.TRACE_INSTANCES) == sorted(TRACE_SPILL_LIMITS)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES + mod.ACTUATOR_INSTANCES + \
        mod.MECHANICS_INSTANCES + mod.CONTACT_INSTANCES + mod.APPLIED_INSTANCES
    assert not any(feat & F_TC for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.TRACE_INSTANCES:   # each is its chain twin of the same precision, kind and features, plus F_TC and nothing else
        assert feat & F_TC and others[COUNTERPART[t]] == (real, dr, feat & ~F_TC)
        assert dr == 1 and feat & F_XF and COUNTERPART[t] in [x for x, *_ in mod.APPLIED_INSTANCES if x.startswith(('f17', 'd17'))]


@pytest.mark.parametrize('tag', sorted(TRACE_SPILL_LIMITS))
def test_trace_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without a trace %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], kernel_resources(COUNTERPART[tag])))
    max_st, max_ld = TRACE_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(TRACE_SPILL_LIMITS))
def test_large_differences_are_explained(tag):
    _, st, ld = kernel_resources(tag)
    _, cst, cld = kernel_resources(COUNTERPART[tag])
    if st - cst > EXPLAIN_ABOVE or ld - cld > EXPLAIN_ABOVE:
        design = open(os.path.join(REPO, 'DESIGN.md')).read()
        assert '`%s`' % tag in design, '%s spills %d / %d bytes more than %s: explain it in DESIGN.md section 5' % (tag, st - cst, ld - cld, COUNTERPART[tag])
