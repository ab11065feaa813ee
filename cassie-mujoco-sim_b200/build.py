"""Builds libcassie_b200.so (sm_90a, H100) in-tree with nvcc.  Used by __graft_entry__.build() and by the Python host module.

The fused step kernel is compiled once per line of csrc/step_instances.inc (precision x kind x features; csrc/step_inst.cu with -D flags), the
instances and the two host-side sources in parallel, then linked into one shared object."""
import os
import re
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, '_obj')
LIB = os.path.join(HERE, 'libcassie_b200.so')
DEPS = [os.path.join(CSRC, f) for f in ('cassie_b200.cu', 'mjcf.cpp', 'step_inst.cu', 'step_kernel.cuh', 'step_core.inl', 'cassie_tree_gen.inc', 'devmodel.h', 'devbuild.h', 'model.h',
                                        'estimator_host.h', 'legacy_stubs.inc', 'step_instances.inc', 'step_select.h', 'env_rows.h', 'raycast.cu', 'raycast.inl', 'camera.cu', 'camera.inl', 'camera_set.cu', 'camera_set.inl', 'reset.cu', 'reset.inl', 'loops.cu', 'loops.inl', 'ik.cu', 'ik.inl')] + [
    os.path.join(HERE, '..', 'include', 'cassie_b200.h'), os.path.join(HERE, '..', 'include', 'cassie_bus.h')]
# (tag, real, kind: 0 plain / 1 extended / 2 plain + estimator, feature bits csrc/devmodel.h F_*) of every step instance, from the tags of
# csrc/step_instances.inc: <f|d><kind digit><feature bits in hex>
with open(os.path.join(CSRC, 'step_instances.inc')) as f:
    STEP_INSTANCES = [(t, 'double' if t[0] == 'd' else 'float', int(t[1]), int(t[2:], 16)) for t in re.findall(r'^STEP_INSTANCE\(([fd][0-2][0-9a-f]+)\)', f.read(), re.M)]


def _twins(bit):
    """the step instances whose highest feature bit is `bit`: the twins that feature added"""
    return [i for i in STEP_INSTANCES if bit <= i[3] < 2 * bit]


# the same instances grouped by the feature they add, one group per resource test (tests/test_*_resources.py); INSTANCES: the model's features only
INSTANCES = [i for i in STEP_INSTANCES if i[3] < 8]
ENV_GEOM_INSTANCES, FRAME_INSTANCES, TERRAIN_INSTANCES, BODY_POS_INSTANCES, ACTUATOR_INSTANCES, MECHANICS_INSTANCES, CONTACT_INSTANCES, APPLIED_INSTANCES, \
    TRACE_INSTANCES, CONTACT_LIST_INSTANCES, SENSOR_INSTANCES = (_twins(1 << b) for b in range(3, 14))
ARCH = ['-gencode', 'arch=compute_90a,code=sm_90a', '-O3', '-lineinfo', '-std=c++17', '-Xcompiler', '-fPIC,-fopenmp'] + os.environ.get('CASSIE_B200_NVCC_EXTRA', '').split()   # extra flags for A/B builds


def nvcc():
    for c in (os.environ.get('NVCC'), '/usr/local/cuda/bin/nvcc', 'nvcc'):
        if c and (os.path.sep not in c or os.path.exists(c)):
            return c
    return 'nvcc'


def _run(cmd, verbose, res=None):
    r = subprocess.run(cmd, capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError('nvcc failed: %s\n%s' % (' '.join(cmd), r.stderr[-6000:]))
    if res:   # the assembler's resource report of a step instance (registers, stack frame, spill bytes per function), kept beside its object
        with open(res, 'w') as f:
            f.write(r.stderr)
    return r.stderr if verbose else ''


def res_path(obj):
    """the resource report written beside a step instance's, the ray kernel's, a camera kernel's, the restore kernel's, the loop-closure kernel's or the
    inverse-kinematics kernel's object file, or None for the other objects."""
    name = os.path.basename(obj)
    return obj[:-2] + '.res' if name.startswith(('step_', 'ray_', 'cam_', 'camset_', 'reset_', 'loops_', 'ik_')) and name.endswith('.o') else None


def build(force=False, verbose=False, out=None):
    lib = out or LIB
    if not out and not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in DEPS):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    ptx = ['-Xptxas', '-v'] if verbose else []
    jobs = []
    for tag, real, dr, feat in STEP_INSTANCES:   # always -Xptxas -v: tests/test_step_resources.py reads the spill counts from csrc/_obj/step_<tag>.res
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DINST_REAL=' + real, '-DINST_DR=%d' % dr, '-DINST_FEAT=%d' % feat, '-DINST_TAG=' + tag, '-c', os.path.join(CSRC, 'step_inst.cu'),
                                           '-o', os.path.join(OBJ, 'step_%s.o' % tag)])
    jobs.append([nvcc()] + ARCH + ptx + ['-c', os.path.join(CSRC, 'cassie_b200.cu'), '-o', os.path.join(OBJ, 'cassie_b200.o')])
    jobs.append([nvcc()] + ARCH + ['-c', os.path.join(CSRC, 'mjcf.cpp'), '-o', os.path.join(OBJ, 'mjcf.o')])
    for real in ('float', 'double'):   # the ray kernel, one object per precision; its report is kept as ray_<real>.res (tests/test_raycast_resources.py)
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DRAY_REAL=' + real, '-c', os.path.join(CSRC, 'raycast.cu'), '-o', os.path.join(OBJ, 'ray_%s.o' % real)])
    for real in ('float', 'double'):   # the camera kernels, likewise; their reports are kept as cam_<real>.res and camset_<real>.res (tests/test_camera_resources.py, test_camera_set_resources.py)
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DCAM_REAL=' + real, '-c', os.path.join(CSRC, 'camera.cu'), '-o', os.path.join(OBJ, 'cam_%s.o' % real)])
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DCAMSET_REAL=' + real, '-c', os.path.join(CSRC, 'camera_set.cu'), '-o', os.path.join(OBJ, 'camset_%s.o' % real)])
    for real in ('float', 'double'):   # the restore kernel, likewise; its report is kept as reset_<real>.res (tests/test_reset_resources.py)
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DRESET_REAL=' + real, '-c', os.path.join(CSRC, 'reset.cu'), '-o', os.path.join(OBJ, 'reset_%s.o' % real)])
    for real in ('float', 'double'):   # the loop-closure kernel, likewise; its report is kept as loops_<real>.res (tests/test_loops_resources.py)
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DLOOPS_REAL=' + real, '-c', os.path.join(CSRC, 'loops.cu'), '-o', os.path.join(OBJ, 'loops_%s.o' % real)])
    for real in ('float', 'double'):   # the inverse-kinematics kernel, likewise; its report is kept as ik_<real>.res (tests/test_ik_resources.py)
        jobs.append([nvcc()] + ARCH + ['-Xptxas', '-v', '-DIK_REAL=' + real, '-c', os.path.join(CSRC, 'ik.cu'), '-o', os.path.join(OBJ, 'ik_%s.o' % real)])
    with ThreadPoolExecutor(max_workers=max(2, min(len(jobs), (os.cpu_count() or 4)))) as ex:
        logs = list(ex.map(lambda c: _run(c, verbose, res_path(c[-1])), jobs))
    if verbose:
        sys.stderr.write(''.join(logs))
    objs = [j[-1] for j in jobs]
    _run([nvcc(), '-gencode', 'arch=compute_90a,code=sm_90a', '-shared', '-Xcompiler', '-fPIC,-fopenmp', '-lgomp', '-o', lib + '.tmp'] + objs, verbose)
    os.replace(lib + '.tmp', lib)   # atomic: a reader never sees a half-written library
    return lib


if __name__ == '__main__':
    print(build(force=True, verbose='-v' in sys.argv, out=sys.argv[sys.argv.index('--out') + 1] if '--out' in sys.argv else None))
