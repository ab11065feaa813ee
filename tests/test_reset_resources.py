"""Register spills of the restore kernel (csrc/reset.cu: cassie_batch_reset_where and the masked cassie_batch_set_state), as the assembler reports them
for sm_90a (no GPU needed).

build.py compiles the kernel once per precision with -Xptxas -v and keeps each report beside its object as csrc/_obj/reset_<real>.res.  Both must stay
free of spills, with the row table read from the parameter bank rather than copied to a stack frame.  The step-kernel instances are not rebuilt for
the restore: their own resource tests hold their reports."""
import os
import re

import pytest

from conftest import REPO

OBJ = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'csrc', '_obj')
_PROPS = re.compile(r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads')


@pytest.mark.parametrize('real', ['float', 'double'])
def test_reset_kernel_has_no_spills(real):
    path = os.path.join(OBJ, 'reset_%s.res' % real)
    if not os.path.exists(path):
        pytest.fail('%s is missing: build the library first (python __graft_entry__.py build)' % path)
    with open(path) as f:
        hits = [m.groups() for m in _PROPS.finditer(f.read()) if 'cassie_reset_kernel' in m.group(1)]
    assert len(hits) == 1, hits
    name, stack, st, ld = hits[0]
    print('%s: %s bytes stack frame, %s bytes spill stores, %s bytes spill loads' % (name, stack, st, ld))
    assert (int(st), int(ld)) == (0, 0)
    assert int(stack) <= 16
