"""Register spills of the step-kernel instances with sensor models (build.py SENSOR_INSTANCES), as the assembler reports them for sm_90a (no GPU
needed), against the F_XF instances they are the F_SN twins of; and the resources of every other instance, which the sensor stage must leave as they
were (tests/golden/step_kernel_resources.json: stack frame, spill stores, spill loads of cassie_step_kernel per instance, CUDA 12.9, before F_SN)."""
import json
import os

import pytest

from conftest import GOLDEN
from test_env_geom_resources import _build_module
from test_step_resources import kernel_resources

F_XF, F_TC, F_CL, F_SN = 1024, 2048, 4096, 8192
# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a, as first built.  Lower them when an edit lowers the spills.
SENSOR_SPILL_LIMITS = {
    'f02404': (96, 116), 'f22404': (104, 132), 'f127c4': (252, 500), 'f127d7': (420, 928), 'd127d7': (1204, 2136), 'f127df': (416, 1012),
    'd127df': (1188, 2212), 'f127ff': (416, 1012), 'd127ff': (1188, 2212),
}
COUNTERPART = {'f02404': 'f0404', 'f22404': 'f2404', 'f127c4': 'f17c4', 'f127d7': 'f17d7', 'd127d7': 'd17d7', 'f127df': 'f17df', 'd127df': 'd17df',
               'f127ff': 'f17ff', 'd127ff': 'd17ff'}
# the sensor stage is its own function (CNOINLINE): a twin may spill at most this many bytes more than its counterpart (stores, loads) and hold a stack
# frame at most this much larger
MAX_EXTRA = (48, 96, 32)


def test_every_sensor_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.SENSOR_INSTANCES) == sorted(SENSOR_SPILL_LIMITS)
    earlier = mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES + mod.ACTUATOR_INSTANCES + \
        mod.MECHANICS_INSTANCES + mod.CONTACT_INSTANCES + mod.APPLIED_INSTANCES + mod.TRACE_INSTANCES + mod.CONTACT_LIST_INSTANCES
    assert not any(feat & F_SN for *_, feat in earlier)
    others = {t: (real, dr, feat) for t, real, dr, feat in earlier}
    for t, real, dr, feat in mod.SENSOR_INSTANCES:   # each is its F_XF instance of the same precision, kind and features, plus F_SN and nothing else
        assert feat & F_SN and others[COUNTERPART[t]] == (real, dr, feat & ~F_SN)
        assert feat & F_XF and not feat & (F_TC | F_CL) and COUNTERPART[t] in [x for x, *_ in mod.APPLIED_INSTANCES]


@pytest.mark.parametrize('tag', sorted(SENSOR_SPILL_LIMITS))
def test_sensor_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    cstack, cst, cld = kernel_resources(COUNTERPART[tag])
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without sensors %s: %d, %d, %d)' % (tag, stack, st, ld, COUNTERPART[tag], cstack, cst, cld))
    max_st, max_ld = SENSOR_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))
    assert st - cst <= MAX_EXTRA[0] and ld - cld <= MAX_EXTRA[1] and stack - cstack <= MAX_EXTRA[2], (tag, COUNTERPART[tag])


def test_other_instances_keep_their_resources():
    """every instance without F_SN: the stack frame and spill bytes it had before the sensor stage was added"""
    want = json.load(open(os.path.join(GOLDEN, 'step_kernel_resources.json')))
    mod = _build_module()
    tags = [t for t, *_, feat in mod.INSTANCES + mod.ENV_GEOM_INSTANCES + mod.FRAME_INSTANCES + mod.TERRAIN_INSTANCES + mod.BODY_POS_INSTANCES +
            mod.ACTUATOR_INSTANCES + mod.MECHANICS_INSTANCES + mod.CONTACT_INSTANCES + mod.APPLIED_INSTANCES + mod.TRACE_INSTANCES + mod.CONTACT_LIST_INSTANCES]
    assert sorted(tags) == sorted(want)
    changed = {t: (want[t], list(kernel_resources(t))) for t in tags if list(kernel_resources(t)) != want[t]}
    assert not changed, changed
