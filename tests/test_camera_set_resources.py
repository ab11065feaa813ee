"""Register spills of every camera-kernel instance, as the assembler reports them for sm_90a (no GPU needed): the one-camera kernel (csrc/camera.cu)
and the camera-set kernel (csrc/camera_set.cu: several cameras, per-environment mounts, geom ids), one instance of each per precision.

build.py keeps each instance's report beside its object as csrc/_obj/cam_<real>.res and camset_<real>.res.  Every function of those reports must be
free of spills; the set kernel's report holds exactly one kernel, whose name does not contain the one-camera kernel's.  The step-kernel instances are
not rebuilt for the cameras (their own resource tests hold their reports)."""
import os
import re

import pytest

from conftest import REPO

OBJ = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'csrc', '_obj')
_PROPS = re.compile(r'Function properties for (\S+)\s*\n\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads')


@pytest.mark.parametrize('obj', ['cam', 'camset'])
@pytest.mark.parametrize('real', ['float', 'double'])
def test_every_camera_kernel_instance_is_spill_free(obj, real):
    path = os.path.join(OBJ, '%s_%s.res' % (obj, real))
    if not os.path.exists(path):
        pytest.fail('%s is missing: build the library first (python __graft_entry__.py build)' % path)
    with open(path) as f:
        props = [m.groups() for m in _PROPS.finditer(f.read())]
    kernels = [p for p in props if ('cassie_camset_kernel' if obj == 'camset' else 'cassie_camera_kernel') in p[0]]
    assert len(kernels) == 1, props
    for name, stack, st, ld in props:
        print('%s: %s bytes stack frame, %s bytes spill stores, %s bytes spill loads' % (name, stack, st, ld))
        assert (int(st), int(ld)) == (0, 0), name
