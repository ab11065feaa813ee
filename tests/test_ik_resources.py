"""Stack frame and spills of the inverse-kinematics kernel (csrc/ik.cu: cassie_batch_solve_ik), as the assembler reports them for sm_90a (no GPU needed).

build.py compiles the kernel once per precision with -Xptxas -v and keeps each report beside its object as csrc/_obj/ik_<real>.res.  The values are those
of the first build; a change to the kernel that moves them shows here.  The step, ray, camera, restore and loop-closure kernels are not rebuilt for it:
their own resource tests hold their reports."""
import os
import re

import pytest

from conftest import REPO

OBJ = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'csrc', '_obj')
_PROPS = re.compile(r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads')
PINNED = {'float': (128, 0, 0), 'double': (232, 0, 0)}   # stack frame, spill stores, spill loads (bytes)


@pytest.mark.parametrize('real', ['float', 'double'])
def test_ik_kernel_keeps_its_stack_and_spills(real):
    path = os.path.join(OBJ, 'ik_%s.res' % real)
    if not os.path.exists(path):
        pytest.fail('%s is missing: build the library first (python __graft_entry__.py build)' % path)
    with open(path) as f:
        hits = [m.groups() for m in _PROPS.finditer(f.read()) if 'cassie_ik_kernel' in m.group(1)]
    assert len(hits) == 1, hits
    name, stack, st, ld = hits[0]
    print('%s: %s bytes stack frame, %s bytes spill stores, %s bytes spill loads' % (name, stack, st, ld))
    assert (int(stack), int(st), int(ld)) == PINNED[real]
