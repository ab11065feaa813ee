"""Register spills of the fused step kernel, as the assembler reports them for sm_90a (no GPU needed).

build.py compiles every step instance with -Xptxas -v and keeps the report beside its object as csrc/_obj/step_<tag>.res.  The kernel runs at the
register file's limit (16 warps per SM, 128 registers per thread), so an edit can push values out to local memory without changing a result; on the
H100 such spills come back from L2 in the middle of dependent chains.  These checks make that visible on a machine without a GPU: each instance's spill
bytes may not exceed what they were when the limits below were last set (zero where zero was reached), and the stack frames are printed."""
import os
import re

import pytest

from conftest import REPO

OBJ = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'csrc', '_obj')
KERNEL = 'cassie_step_kernel'

# (spill store bytes, spill load bytes) of cassie_step_kernel per instance, CUDA 12.9, sm_90a.  Lower them when an edit lowers the spills.
# f*0 / f*2 / f*4 / f*5 / f*7: feature sets (none, height field, boxes, boxes + free body, all); f0x plain, f1x extended, f2x plain + estimator.
SPILL_LIMITS = {
    'f00': (0, 0), 'f02': (156, 204), 'f04': (96, 112), 'f05': (140, 188), 'f07': (244, 364),
    'f20': (16, 20), 'f22': (148, 208), 'f24': (112, 136), 'f25': (148, 208), 'f27': (252, 380),
    'f10': (140, 200), 'f12': (292, 560), 'f14': (244, 456), 'f15': (320, 612), 'f17': (432, 952),
    'd07': (964, 1372), 'd17': (1188, 2140), 'd27': (976, 1388),
}

_PROPS = re.compile(r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads')


def resources(tag):
    """{function: (stack frame, spill stores, spill loads)} from the assembler report of instance `tag`."""
    path = os.path.join(OBJ, 'step_%s.res' % tag)
    if not os.path.exists(path):
        pytest.fail('%s is missing: build the library first (python __graft_entry__.py build)' % path)
    with open(path) as f:
        return {m.group(1): tuple(int(m.group(i)) for i in (2, 3, 4)) for m in _PROPS.finditer(f.read())}


def kernel_resources(tag):
    hits = [v for k, v in resources(tag).items() if KERNEL in k]
    assert len(hits) == 1, ('expected one %s in the report of %s' % (KERNEL, tag), hits)
    return hits[0]


def test_parse_report():
    txt = ("ptxas info    : Function properties for _ZN6cassie18cassie_step_kernelIfLi0ELi4EEEvPKNS_8DevModelIT_EENS_9EnvArraysIS2_EEii\n"
           "    272 bytes stack frame, 96 bytes spill stores, 112 bytes spill loads\n")
    m = _PROPS.search(txt)
    assert m and KERNEL in m.group(1) and (m.group(2), m.group(3), m.group(4)) == ('272', '96', '112')


def test_every_instance_is_listed():
    import importlib.util
    spec = importlib.util.spec_from_file_location('_cassie_b200_build', os.path.join(REPO, 'cassie-mujoco-sim_b200', 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    assert sorted(t for t, *_ in mod.INSTANCES) == sorted(SPILL_LIMITS)


@pytest.mark.parametrize('tag', sorted(SPILL_LIMITS))
def test_step_kernel_spills(tag):
    stack, st, ld = kernel_resources(tag)
    print('%s: %d bytes stack frame, %d bytes spill stores, %d bytes spill loads' % (tag, stack, st, ld))
    max_st, max_ld = SPILL_LIMITS[tag]
    assert st <= max_st and ld <= max_ld, ('%s spills more than before: %d / %d bytes stored / loaded, limit %d / %d' % (tag, st, ld, max_st, max_ld))
