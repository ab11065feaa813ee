"""Register spills of the step-kernel instances that fill frame rows (build.py FRAME_INSTANCES), as the assembler reports them for sm_90a (no GPU
needed), and the frame stages' absence from every other instance: the shipped and per-environment-geom instances keep their resource reports."""
import pytest

from test_env_geom_resources import ENV_GEOM_SPILL_LIMITS, _build_module
from test_step_resources import SPILL_LIMITS, kernel_resources

# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a.  Lower them when an edit lowers the spills.
FRAME_SPILL_LIMITS = {
    'f114': (272, 444), 'f117': (432, 868), 'd117': (1140, 2016),
    'f11c': (244, 396), 'f11f': (400, 792), 'd11f': (1148, 2108),
}
COUNTERPART = {'f114': 'f14', 'f117': 'f17', 'd117': 'd17', 'f11c': 'f1c', 'f11f': 'f1f', 'd11f': 'd1f'}
# stack frame, spill stores, spill loads of the instances without frame stages, as they were before the frame stages were added (CUDA 12.9)
UNCHANGED = {
    'f00': (32, 0, 0), 'f10': (368, 140, 200), 'f02': (152, 156, 204), 'f12': (480, 292, 560), 'f04': (272, 96, 112), 'f14': (560, 244, 456),
    'f05': (320, 140, 188), 'f15': (640, 320, 612), 'f07': (400, 244, 364), 'f17': (704, 432, 952), 'd07': (896, 964, 1372), 'd17': (1072, 1188, 2140),
    'f20': (240, 16, 20), 'f22': (352, 148, 208), 'f24': (432, 112, 136), 'f25': (496, 148, 208), 'f27': (560, 252, 380), 'd27': (928, 976, 1388),
    'f0c': (224, 32, 40), 'f1c': (512, 188, 292), 'f2c': (384, 44, 60), 'f0f': (416, 256, 400), 'f1f': (720, 444, 940), 'f2f': (560, 264, 416),
    'd0f': (896, 972, 1392), 'd1f': (1104, 1220, 2152), 'd2f': (928, 984, 1408),
}


def test_every_frame_instance_is_listed():
    mod = _build_module()
    assert sorted(t for t, *_ in mod.FRAME_INSTANCES) == sorted(FRAME_SPILL_LIMITS)
    assert all(feat & 16 and dr == 1 for _, _, dr, feat in mod.FRAME_INSTANCES)
    assert not any(feat & 16 for *_, feat in mod.INSTANCES + mod.ENV_GEOM_INSTANCES)
    others = {t: (real, dr, feat) for t, real, dr, feat in mod.INSTANCES + mod.ENV_GEOM_INSTANCES}
    for t, real, dr, feat in mod.FRAME_INSTANCES:   # each has a counterpart without frames of the same precision, kind and features
        assert others[COUNTERPART[t]] == (real, dr, feat & ~16)
    assert sorted(UNCHANGED) == sorted(list(SPILL_LIMITS) + list(ENV_GEOM_SPILL_LIMITS))


@pytest.mark.parametrize('tag', sorted(FRAME_SPILL_LIMITS))
def test_frame_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads (without frames %s: %s)' % (tag, stack, st, ld, COUNTERPART[tag], UNCHANGED[COUNTERPART[tag]]))
    max_st, max_ld = FRAME_SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))


@pytest.mark.parametrize('tag', sorted(UNCHANGED))
def test_instances_without_frames_are_unchanged(tag):
    assert kernel_resources(tag) == UNCHANGED[tag]
