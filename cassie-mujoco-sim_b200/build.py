"""Builds libcassie_b200.so (sm_90a, H100) in-tree with nvcc.  Used by __graft_entry__.build() and by the Python host module.

The fused step kernel is compiled once per instance (precision x plain / extended x model features; csrc/step_inst.cu with -D flags), the
instances and the two host-side sources in parallel, then linked into one shared object."""
import os
import subprocess
import sys
from concurrent.futures import ThreadPoolExecutor

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, 'csrc')
OBJ = os.path.join(CSRC, '_obj')
LIB = os.path.join(HERE, 'libcassie_b200.so')
DEPS = [os.path.join(CSRC, f) for f in ('cassie_b200.cu', 'mjcf.cpp', 'step_inst.cu', 'step_kernel.cuh', 'step_core.inl', 'cassie_tree_gen.inc', 'devmodel.h', 'devbuild.h', 'model.h',
                                        'estimator_host.h', 'legacy_stubs.inc', 'raycast.cu', 'raycast.inl', 'camera.cu', 'camera.inl', 'camera_set.cu', 'camera_set.inl', 'reset.cu', 'reset.inl')] + [
    os.path.join(HERE, '..', 'include', 'cassie_b200.h'), os.path.join(HERE, '..', 'include', 'cassie_bus.h')]
# (tag, real, instance: 0 plain / 1 extended / 2 plain + estimator, feature set): features 1 = extra free body, 2 = height field, 4 = box geoms (csrc/devmodel.h F_*)
INSTANCES = [('f00', 'float', 0, 0), ('f10', 'float', 1, 0), ('f02', 'float', 0, 2), ('f12', 'float', 1, 2), ('f04', 'float', 0, 4), ('f14', 'float', 1, 4), ('f05', 'float', 0, 5), ('f15', 'float', 1, 5),
             ('f07', 'float', 0, 7), ('f17', 'float', 1, 7), ('d07', 'double', 0, 7), ('d17', 'double', 1, 7),
             ('f20', 'float', 2, 0), ('f22', 'float', 2, 2), ('f24', 'float', 2, 4), ('f25', 'float', 2, 5), ('f27', 'float', 2, 7), ('d27', 'double', 2, 7)]
# the same kernel with the static geoms' placement read from per-environment rows (feature 8 = F_EG; cassie_batch_set_env_geom_pose): boxes (also for
# models without boxes, floor tilt only) or every feature, in each instance kind; the tag's last digit is the feature set in hex
ENV_GEOM_INSTANCES = [('f0c', 'float', 0, 12), ('f1c', 'float', 1, 12), ('f2c', 'float', 2, 12), ('f0f', 'float', 0, 15), ('f1f', 'float', 1, 15), ('f2f', 'float', 2, 15),
                      ('d0f', 'double', 0, 15), ('d1f', 'double', 1, 15), ('d2f', 'double', 2, 15)]
# the extended kernel with frame rows (feature 16 = F_FR; cassie_batch_set_frames): boxes or every feature, without and with the per-environment static
# geoms; tag = precision, instance kind, feature set in hex
FRAME_INSTANCES = [('f114', 'float', 1, 20), ('f117', 'float', 1, 23), ('d117', 'double', 1, 23),
                   ('f11c', 'float', 1, 28), ('f11f', 'float', 1, 31), ('d11f', 'double', 1, 31)]
# every feature with the per-environment static geoms and per-environment terrain (feature 32 = F_TR; cassie_batch_set_env_hfield): the bank entry and the
# height field's size come from per-environment rows; in each instance kind, and the extended kernel with frame rows; tag = precision, kind, features in hex
TERRAIN_INSTANCES = [('f02f', 'float', 0, 47), ('f12f', 'float', 1, 47), ('f22f', 'float', 2, 47), ('d02f', 'double', 0, 47), ('d12f', 'double', 1, 47), ('d22f', 'double', 2, 47),
                     ('f13f', 'float', 1, 63), ('d13f', 'double', 1, 63)]
# the extended kernel with per-environment body offsets (feature 64 = F_BP; cassie_batch_set_env_body_pos): each differs from its counterpart (f14, f117 /
# d117, f11f / d11f, f13f / d13f) by F_BP only; tag = precision, kind, features in hex
BODY_POS_INSTANCES = [('f144', 'float', 1, 68), ('f157', 'float', 1, 87), ('d157', 'double', 1, 87), ('f15f', 'float', 1, 95), ('d15f', 'double', 1, 95),
                      ('f17f', 'float', 1, 127), ('d17f', 'double', 1, 127)]
# the extended kernel with per-environment actuators (feature 128 = F_AC; cassie_batch_set_env_actuators), always with body-offset rows (a batch with
# actuator rows carries offset rows holding the model's values when it has no others): each is the F_AC twin of one BODY_POS_INSTANCES entry (f144,
# f157 / d157, f15f / d15f, f17f / d17f); tag = precision, kind, features in hex
ACTUATOR_INSTANCES = [('f1c4', 'float', 1, 196), ('f1d7', 'float', 1, 215), ('d1d7', 'double', 1, 215), ('f1df', 'float', 1, 223), ('d1df', 'double', 1, 223),
                      ('f1ff', 'float', 1, 255), ('d1ff', 'double', 1, 255)]
# the extended kernel with per-environment mechanics (feature 256 = F_MC; cassie_batch_set_env_mechanics: link inertia, rotor armature, hinge springs), always
# with actuator rows (a batch with mechanics rows carries actuator rows holding the model's values when it has no others, and offset rows through them):
# each is the F_MC twin of one ACTUATOR_INSTANCES entry (f1c4, f1d7 / d1d7, f1df / d1df, f1ff / d1ff); tag = precision, kind, features in hex
MECHANICS_INSTANCES = [('f11c4', 'float', 1, 452), ('f11d7', 'float', 1, 471), ('d11d7', 'double', 1, 471), ('f11df', 'float', 1, 479), ('d11df', 'double', 1, 479),
                       ('f11ff', 'float', 1, 511), ('d11ff', 'double', 1, 511)]
# the extended kernel with per-environment contact softness (feature 512 = F_CT; cassie_batch_set_env_contact: solref, solimp, solmix per collision geom),
# always with mechanics rows (a batch with contact rows carries mechanics rows holding the model's values when it has no others, and actuator and offset
# rows through them): each is the F_CT twin of one MECHANICS_INSTANCES entry (f11c4, f11d7 / d11d7, f11df / d11df, f11ff / d11ff); tag = precision,
# kind, features in hex
CONTACT_INSTANCES = [('f13c4', 'float', 1, 964), ('f13d7', 'float', 1, 983), ('d13d7', 'double', 1, 983), ('f13df', 'float', 1, 991), ('d13df', 'double', 1, 991),
                     ('f13ff', 'float', 1, 1023), ('d13ff', 'double', 1, 1023)]
# per-environment applied forces (feature 1024 = F_XF; cassie_batch_set_applied_forces: xfrc_applied per body, qfrc_applied per dof).  The push workload
# runs the plain kinds: f0404 / f2404 are the F_XF twins of f04 / f24 and run where those would.  Any other batch with applied rows runs the extended
# kernel, which carries contact rows holding the model's values (and mechanics, actuator and offset rows through them): the chain twins, each the F_XF
# twin of one CONTACT_INSTANCES entry (f13c4, f13d7 / d13d7, f13df / d13df, f13ff / d13ff); tag = precision, kind, features in hex
APPLIED_INSTANCES = [('f0404', 'float', 0, 1028), ('f2404', 'float', 2, 1028),
                     ('f17c4', 'float', 1, 1988), ('f17d7', 'float', 1, 2007), ('d17d7', 'double', 1, 2007), ('f17df', 'float', 1, 2015), ('d17df', 'double', 1, 2015),
                     ('f17ff', 'float', 1, 2047), ('d17ff', 'double', 1, 2047)]
# per-tick traces (feature 2048 = F_TC; cassie_batch_set_trace): every tick of a step launch stores the traced qpos / qvel / observation / derived-quantity
# / frame columns into its slot of the trace rows.  Any batch with a trace runs one of these, each the F_TC twin of one chain twin of APPLIED_INSTANCES
# (f17c4, f17d7 / d17d7, f17df / d17df, f17ff / d17ff), with the model-valued applied, contact, mechanics, actuator and offset rows the chain twins read;
# tag = precision, kind, features in hex
TRACE_INSTANCES = [('f1fc4', 'float', 1, 4036), ('f1fd7', 'float', 1, 4055), ('d1fd7', 'double', 1, 4055), ('f1fdf', 'float', 1, 4063), ('d1fdf', 'double', 1, 4063),
                   ('f1fff', 'float', 1, 4095), ('d1fff', 'double', 1, 4095)]
# contact lists (feature 4096 = F_CL; cassie_batch_enable_contacts): the last sub-step of a step or forward launch stores MuJoCo's contact list and
# mj_contactForce into the contact-list rows.  Any batch with contact lists runs one of these, each the F_CL twin of one F_FR chain twin of
# APPLIED_INSTANCES (f17d7 / d17d7, f17df / d17df, f17ff / d17ff), with the model-valued applied, contact, mechanics, actuator and offset rows the chain
# twins read; tag = precision, kind, features in hex
CONTACT_LIST_INSTANCES = [('f117d7', 'float', 1, 6103), ('d117d7', 'double', 1, 6103), ('f117df', 'float', 1, 6111), ('d117df', 'double', 1, 6111),
                          ('f117ff', 'float', 1, 6143), ('d117ff', 'double', 1, 6143)]
# sensor models (feature 8192 = F_SN; cassie_batch_set_env_sensors): encoder offsets and noise, IMU mount, bias and noise applied to the controller stage's
# copy of the sensordata every tick.  The plain twins f02404 / f22404 (F_SN | F_XF | F_BOX) run where f04 / f24 / f0404 / f2404 would, with zeroed applied
# rows when the batch has none; any other batch with sensor rows runs the F_SN twin of the F_XF chain twin its rule picks (f17c4, f17d7 / d17d7, f17df /
# d17df, f17ff / d17ff), with the model-valued applied, contact, mechanics, actuator and offset rows the chain twins read; tag = precision, kind, features in hex
SENSOR_INSTANCES = [('f02404', 'float', 0, 9220), ('f22404', 'float', 2, 9220),
                    ('f127c4', 'float', 1, 10180), ('f127d7', 'float', 1, 10199), ('d127d7', 'double', 1, 10199), ('f127df', 'float', 1, 10207), ('d127df', 'double', 1, 10207),
                    ('f127ff', 'float', 1, 10239), ('d127ff', 'double', 1, 10239)]
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
    """the resource report written beside a step instance's, the ray kernel's, a camera kernel's or the restore kernel's object file, or None for the other objects."""
    name = os.path.basename(obj)
    return obj[:-2] + '.res' if name.startswith(('step_', 'ray_', 'cam_', 'camset_', 'reset_')) and name.endswith('.o') else None


def build(force=False, verbose=False, out=None):
    lib = out or LIB
    if not out and not force and os.path.exists(LIB) and all(os.path.getmtime(LIB) >= os.path.getmtime(d) for d in DEPS):
        return LIB
    os.makedirs(OBJ, exist_ok=True)
    ptx = ['-Xptxas', '-v'] if verbose else []
    jobs = []
    for tag, real, dr, feat in INSTANCES + ENV_GEOM_INSTANCES + FRAME_INSTANCES + TERRAIN_INSTANCES + BODY_POS_INSTANCES + ACTUATOR_INSTANCES + MECHANICS_INSTANCES + CONTACT_INSTANCES + APPLIED_INSTANCES + TRACE_INSTANCES + CONTACT_LIST_INSTANCES + SENSOR_INSTANCES:   # always -Xptxas -v: tests/test_step_resources.py reads the spill counts from csrc/_obj/step_<tag>.res
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
