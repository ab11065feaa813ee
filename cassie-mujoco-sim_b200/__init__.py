"""cassie-mujoco-sim_b200 -- Python host side of the H100-native (sm_90a) batched Cassie stepper.

Mirrors the reference's Python surface for the one path this repo accelerates
(example/cassiemujoco.py:31-173 of the original project: CassieSim.step_pd / qpos / qvel / set_qpos / apply_force ...)
on top of the C-ABI in include/cassie_b200.h, and adds CassieBatch for the batched entry points.
There is no CPU fallback: loading fails loudly if the CUDA library is missing, and cassie_batch_init fails if no GPU is visible.
"""
import ctypes as C
import os

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, 'libcassie_b200.so')
MODEL_DIR = os.path.join(_HERE, 'models')
FP32, FP64 = 0, 1
LINE_MAX = 6   # the longest torque delay in control ticks (the delay line's length, csrc/devmodel.h AC_MAXDELAY)
NU = 10   # motors: every supported model has Cassie's ten (csrc/devmodel.h MU), in the model's actuator order
PD_WIDTH, OBS_WIDTH, AUX_WIDTH, EST_WIDTH = 52, 112, 64, 16
# one frame's slot of a frame row (CASSIE_FRAME_* in include/cassie_b200.h) and the frame kinds of set_frames
FRAME_WIDTH, FRAME_BODY, FRAME_SITE, FRAME_MAX = 20, 0, 1, 64
IK_MAX, IK_TARGET_WIDTH, IK_SLOT, IK_WORLD, IK_ROOT = 4, 16, 8, 0, 1   # include/cassie_b200.h CASSIE_IK_*
IK_STATUS = ('pos_residual', 'ori_residual', 'loop_residual', 'iterations', 'outcome', 'jeq_qvel', 'vel_residual', 'at_bound')
FRAME = dict(pos=slice(0, 3), quat=slice(3, 7), vel=slice(7, 13), cfrc=slice(13, 19))
# dynamics row (include/cassie_b200.h CASSIE_DYN_*): M [40][40], bias [40], connect rows [12][40], their errors [12], centre-of-mass offset [3]
DYN_WIDTH, DYN_COLS = 2144, 40
# terrain rays (include/cassie_b200.h CASSIE_RAY_*): frame kinds of set_rays, and per ray and environment distance (-1: none), world z of the hit (of
# the ray's end point when none), static geom slot (-1: none), pad
RAY_HEADING, RAY_ROOT, RAY_WORLD, RAY_MAX, RAY_SLOT = 0, 1, 2, 1024, 4
RAY_FRAMES = dict(heading=RAY_HEADING, root=RAY_ROOT, world=RAY_WORLD)
# depth cameras (include/cassie_b200.h CASSIE_CAM_*): largest image side, cameras per set, reals per per-environment mount slot (pos[3], quat[4],
# fovy in degrees)
CAM_MAXDIM = 256
CAM_MAX = 4
CAMENV_SLOT = 8
DYN = dict(M=slice(0, 1600), bias=slice(1600, 1640), J_eq=slice(1640, 2120), eq_err=slice(2120, 2132), rcm=slice(2132, 2135))
# inverse row (include/cassie_b200.h CASSIE_INV_*): qfrc_inverse [40], qfrc_constraint [40] (column = dof as in DYN), then the row count, the contacts with
# rows and the contacts dropped at the capacities, as reals; padded to 96.  The input rows ('inv_qacc') are qvel-wide, column = dof
INV_WIDTH, INV_COLS = 96, 40
INV = dict(qfrc_inverse=slice(0, 40), qfrc_constraint=slice(40, 80), nefc=80, ncon=81, dropped=82)
# acceleration row (include/cassie_b200.h CASSIE_ACC_*): qacc [40] (column = dof), then per frame f a slot of ACC_SLOT at ACC_QCOLS + ACC_SLOT f holding
# cacc [6] (com-based [angular; linear]) and 2 pad.  ACC['qacc'] slices the row, ACC['cacc'] a frame's slot
ACC_QCOLS, ACC_SLOT = 40, 8
ACC = dict(qacc=slice(0, 40), cacc=slice(0, 6))


def acc_width(nframes):
    """width of an acceleration row with `nframes` frames"""
    return ACC_QCOLS + ACC_SLOT * nframes
# slices of a derived-quantity row (CASSIE_AUX_* in include/cassie_b200.h)
AUX = dict(foot_force=slice(0, 12), toe_force=slice(12, 18), heel_force=slice(18, 24), foot_pos=slice(24, 30), foot_vel=slice(30, 42),
           cm_pos=slice(42, 45), cm_vel=slice(45, 48), angmom=slice(48, 51), obstacle=51, self_collision=52, group_mask=53, ncon=54)
# per-tick trace sources (include/cassie_b200.h CASSIE_TRACE_*): CassieBatch.set_trace columns are (source, column) pairs, columns as OBS / AUX / FRAME slice
# the rows (a frame column is frame * FRAME_WIDTH + an offset of FRAME)
TRACE_QPOS, TRACE_QVEL, TRACE_OBS, TRACE_AUX, TRACE_FRAME, TRACE_MAX = 0, 1, 2, 3, 4, 64
# contact-list row layout (include/cassie_b200.h CASSIE_CON_*): a header of CON_HEAD reals (listed, found, dropped), then CON_MAX slots of CON_SLOT reals;
# CON slices a slot
CON_HEAD, CON_SLOT, CON_MAX, CON_WIDTH = 8, 24, 12, 296
CON = dict(geom1=0, geom2=1, dim=2, dist=3, pos=slice(4, 7), frame=slice(7, 16), force=slice(16, 22), mu=22, efc=23)
# observation row layout (cassie_batch_get_obs)
OBS = dict(motor_pos=slice(0, 10), motor_vel=slice(10, 20), motor_torque=slice(20, 30), joint_pos=slice(30, 36), joint_vel=slice(36, 42),
           quat=slice(42, 46), gyro=slice(46, 49), accel=slice(49, 52), mag=slice(52, 55), time=55,
           # decoded estimator (state_output_step): stateless part ...
           est_accel=slice(56, 59), left_foot=slice(60, 73), right_foot=slice(73, 86), est_quat=slice(86, 90),
           # ... and, once the in-kernel estimator is on, the force model and the filters
           est_position=slice(96, 99), est_velocity=slice(99, 102), est_external_force=slice(102, 105), est_terrain_height=105,
           est_left_toe_force=slice(106, 109), est_right_toe_force=slice(109, 112))


# ---------------------------------------------------------------- ctypes mirrors of the bus structs (include/cassie_bus.h)
class pd_motor_in_t(C.Structure):
    _fields_ = [(n, C.c_double * 5) for n in ('torque', 'pTarget', 'dTarget', 'pGain', 'dGain')]


class pd_task_in_t(C.Structure):
    _fields_ = [(n, C.c_double * 6) for n in ('torque', 'pTarget', 'dTarget', 'pGain', 'dGain')]


class pd_leg_in_t(C.Structure):
    _fields_ = [('taskPd', pd_task_in_t), ('motorPd', pd_motor_in_t)]


class pd_in_t(C.Structure):
    _fields_ = [('leftLeg', pd_leg_in_t), ('rightLeg', pd_leg_in_t), ('telemetry', C.c_double * 9)]


class state_battery_out_t(C.Structure):
    _fields_ = [('stateOfCharge', C.c_double), ('current', C.c_double)]


class state_foot_out_t(C.Structure):
    _fields_ = [('position', C.c_double * 3), ('orientation', C.c_double * 4), ('footRotationalVelocity', C.c_double * 3),
                ('footTranslationalVelocity', C.c_double * 3), ('toeForce', C.c_double * 3), ('heelForce', C.c_double * 3)]


class state_joint_out_t(C.Structure):
    _fields_ = [('position', C.c_double * 6), ('velocity', C.c_double * 6)]


class state_motor_out_t(C.Structure):
    _fields_ = [('position', C.c_double * 10), ('velocity', C.c_double * 10), ('torque', C.c_double * 10)]


class state_pelvis_out_t(C.Structure):
    _fields_ = [('position', C.c_double * 3), ('orientation', C.c_double * 4), ('rotationalVelocity', C.c_double * 3),
                ('translationalVelocity', C.c_double * 3), ('translationalAcceleration', C.c_double * 3),
                ('externalMoment', C.c_double * 3), ('externalForce', C.c_double * 3)]


class state_radio_out_t(C.Structure):
    _fields_ = [('channel', C.c_double * 16), ('signalGood', C.c_bool)]


class state_terrain_out_t(C.Structure):
    _fields_ = [('height', C.c_double), ('slope', C.c_double * 2)]


class state_out_t(C.Structure):
    _fields_ = [('pelvis', state_pelvis_out_t), ('leftFoot', state_foot_out_t), ('rightFoot', state_foot_out_t),
                ('terrain', state_terrain_out_t), ('motor', state_motor_out_t), ('joint', state_joint_out_t),
                ('radio', state_radio_out_t), ('battery', state_battery_out_t)]


assert C.sizeof(pd_in_t) == 952 and C.sizeof(state_out_t) == 992

_lib = None


def build(force=False, verbose=False):
    """compile libcassie_b200.so in-tree (nvcc, sm_90a)."""
    import importlib.util
    spec = importlib.util.spec_from_file_location('_cassie_b200_build', os.path.join(_HERE, 'build.py'))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod.build(force=force, verbose=verbose)


def lib():
    """the loaded C-ABI library; raises if it has not been built (no fallback path exists)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError('libcassie_b200.so is missing: run `python __graft_entry__.py build` (nvcc, sm_90a). '
                           'The batched stepper has no CPU fallback.')
    L = C.CDLL(LIB_PATH)
    vp, ci, cd = C.c_void_p, C.c_int, C.POINTER(C.c_double)
    L.cassie_b200_last_error.restype = C.c_char_p
    L.cassie_batch_init.restype = vp
    L.cassie_batch_init.argtypes = [C.c_char_p, ci, ci, ci]
    L.cassie_batch_free.argtypes = [vp]
    for n in ('cassie_batch_nenv', 'cassie_batch_nq', 'cassie_batch_nv', 'cassie_batch_precision'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = ci
    L.cassie_batch_launch_count.argtypes = [vp]
    L.cassie_batch_launch_count.restype = C.c_long
    L.cassie_batch_reset.argtypes = [vp, C.c_void_p]
    L.cassie_sim_step_pd_batch.argtypes = [vp, C.c_void_p, C.c_void_p]
    L.cassie_batch_set_pd.argtypes = [vp, cd]
    L.cassie_batch_step.argtypes = [vp, ci]
    for n in ('cassie_batch_sync', 'cassie_batch_forward', 'cassie_batch_clear_forces', 'cassie_batch_integrate_pos'):
        getattr(L, n).argtypes = [vp]
    for n in ('cassie_batch_get_qpos', 'cassie_batch_set_qpos', 'cassie_batch_get_qvel', 'cassie_batch_set_qvel', 'cassie_batch_get_time',
              'cassie_batch_get_obs'):
        getattr(L, n).argtypes = [vp, cd]
    L.cassie_batch_apply_force.argtypes = [vp, cd, C.c_char_p]
    L.cassie_batch_apply_force.restype = ci
    L.cassie_batch_set_hfielddata.argtypes = [vp, C.POINTER(C.c_float), ci]
    L.cassie_batch_set_hfielddata.restype = ci
    for n in ('cassie_batch_hfield_nrow', 'cassie_batch_hfield_ncol'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = ci
    L.cassie_batch_device_ptr.argtypes = [vp, C.c_char_p]
    L.cassie_batch_device_ptr.restype = vp
    L.cassie_batch_set_stream.argtypes = [vp, vp]
    L.cassie_batch_get_stream.argtypes = [vp]
    L.cassie_batch_get_stream.restype = vp
    L.cassie_batch_get_counters.argtypes = [vp, C.POINTER(ci)]
    L.cassie_batch_debug_dump.argtypes = [vp, ci, cd, ci]
    L.cassie_batch_debug_dump.restype = ci
    # legacy verbs
    L.cassie_mujoco_init.argtypes = [C.c_char_p]
    L.cassie_mujoco_init.restype = C.c_bool
    L.cassie_sim_init.argtypes = [C.c_char_p, C.c_bool]
    L.cassie_sim_init.restype = vp
    L.cassie_sim_free.argtypes = [vp]
    L.cassie_sim_step_pd.argtypes = [vp, C.POINTER(state_out_t), C.POINTER(pd_in_t)]
    for n in ('cassie_sim_time', 'cassie_sim_qpos', 'cassie_sim_qvel', 'cassie_sim_timestep', 'cassie_state_time', 'cassie_state_qpos', 'cassie_state_qvel'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = cd
    L.cassie_sim_step.argtypes = [vp, vp, vp]
    L.cassie_sim_step_pd_no2khz.argtypes = [vp, C.POINTER(state_out_t), C.POINTER(pd_in_t)]
    L.cassie_sim_set_timestep.argtypes = [vp, C.c_double]
    L.cassie_sim_forward.argtypes = [vp]
    L.cassie_sim_forward.restype = ci
    for n in ('cassie_sim_hold', 'cassie_sim_release', 'cassie_state_free'):
        getattr(L, n).argtypes = [vp]
    for n in ('cassie_get_state', 'cassie_set_state', 'cassie_sim_copy', 'cassie_state_copy'):
        getattr(L, n).argtypes = [vp, vp]
    L.cassie_state_alloc.restype = vp
    L.cassie_sim_duplicate.argtypes = [vp]
    L.cassie_sim_duplicate.restype = vp
    for n in ('cassie_sim_nv', 'cassie_sim_nq'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = ci
    L.cassie_sim_apply_force.argtypes = [vp, cd, C.c_char_p]
    L.cassie_sim_clear_forces.argtypes = [vp]
    L.cassie_sim_full_reset.argtypes = [vp]
    L.cassie_sim_radio.argtypes = [vp, cd]
    for n in ('cassie_batch_enable_aux',):
        getattr(L, n).argtypes = [vp, ci]
        getattr(L, n).restype = ci
    L.cassie_batch_enable_estimator_forces.argtypes = [vp, ci]
    L.cassie_batch_enable_estimator_forces.restype = ci
    L.cassie_batch_enable_estimator_filter.argtypes = [vp, ci]
    L.cassie_batch_enable_estimator_filter.restype = ci
    L.cassie_batch_reset_estimator.argtypes = [vp, C.c_void_p]
    L.cassie_batch_reset_estimator.restype = ci
    L.cassie_batch_enable_estimator_device.argtypes = [vp, ci]
    L.cassie_batch_enable_estimator_device.restype = ci
    L.cassie_batch_get_estimator.argtypes = [vp, cd]
    L.cassie_batch_get_estimator.restype = ci
    L.cassie_batch_set_pd_gait.argtypes = [vp, cd, cd, cd]
    L.cassie_batch_set_pd_gait.restype = ci
    L.cassie_batch_set_task_pd.argtypes = [vp, cd]
    L.cassie_batch_set_task_pd.restype = ci
    L.cassie_batch_get_aux.argtypes = [vp, cd]
    L.cassie_batch_get_aux.restype = ci
    L.cassie_batch_query.argtypes = [vp]
    L.cassie_batch_query.restype = ci
    L.cassie_batch_row_width.argtypes = [vp, C.c_char_p]
    L.cassie_batch_row_width.restype = ci
    for n in ('cassie_batch_nbody', 'cassie_batch_ngeom'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = ci
    for what in ('body_mass', 'body_ipos', 'dof_damping', 'geom_friction'):
        for op in ('set', 'get'):
            f = getattr(L, 'cassie_batch_%s_%s' % (op, what))
            f.argtypes = [vp, cd]
            f.restype = ci
    L.cassie_batch_set_const.argtypes = [vp, C.c_void_p, ci]
    L.cassie_batch_set_const.restype = ci
    L.cassie_batch_set_geom_pose.argtypes = [vp, C.c_char_p, cd, cd, cd]
    L.cassie_batch_set_geom_pose.restype = ci
    L.cassie_batch_set_env_geom_pose.argtypes = [vp, C.c_char_p, cd, cd, cd, C.c_void_p]
    L.cassie_batch_set_env_geom_pose.restype = ci
    L.cassie_batch_get_env_geom_pose.argtypes = [vp, C.c_char_p, cd, cd, cd]
    L.cassie_batch_get_env_geom_pose.restype = ci
    L.cassie_batch_clear_env_geom_poses.argtypes = [vp]
    L.cassie_batch_clear_env_geom_poses.restype = ci
    L.cassie_batch_set_env_hfield.argtypes = [vp, C.POINTER(ci), cd, cd, C.c_void_p]
    L.cassie_batch_get_env_hfield.argtypes = [vp, C.POINTER(ci), cd, cd]
    L.cassie_batch_clear_env_hfield.argtypes = [vp]
    L.cassie_batch_set_hfield_size.argtypes = L.cassie_batch_get_hfield_size.argtypes = [vp, cd]
    for n in ('set_env_hfield', 'get_env_hfield', 'clear_env_hfield', 'set_hfield_size', 'get_hfield_size'):
        getattr(L, 'cassie_batch_' + n).restype = ci
    L.cassie_sim_get_hfield_size.argtypes = [vp]
    L.cassie_sim_get_hfield_size.restype = cd
    L.cassie_sim_set_hfield_size.argtypes = [vp, C.c_double * 4]
    L.cassie_sim_params.argtypes = [vp, C.POINTER(ci)]
    for n in ('cassie_sim_dof_damping', 'cassie_sim_body_mass', 'cassie_sim_body_ipos', 'cassie_sim_geom_friction'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = cd
    for n in ('cassie_sim_set_dof_damping', 'cassie_sim_set_body_mass', 'cassie_sim_set_body_ipos', 'cassie_sim_set_geom_friction'):
        getattr(L, n).argtypes = [vp, cd]
        getattr(L, n).restype = None
    L.cassie_batch_set_env_body_pos.argtypes = [vp, cd, C.c_void_p]
    L.cassie_batch_get_env_body_pos.argtypes = [vp, cd]
    L.cassie_batch_clear_env_body_pos.argtypes = [vp]
    for n in ('set_env_body_pos', 'get_env_body_pos', 'clear_env_body_pos'):
        getattr(L, 'cassie_batch_' + n).restype = ci
    for n in ('cassie_sim_set_dof_name_damping', 'cassie_sim_set_body_name_ipos', 'cassie_sim_set_geom_name_friction', 'cassie_sim_set_body_name_pos'):
        getattr(L, n).argtypes = [vp, C.c_char_p, cd]
        getattr(L, n).restype = None
    for n in ('cassie_sim_get_dof_name_damping', 'cassie_sim_get_body_name_ipos', 'cassie_sim_get_geom_name_friction', 'cassie_sim_get_body_name_pos'):
        getattr(L, n).argtypes = [vp, C.c_char_p]
        getattr(L, n).restype = cd
    L.cassie_sim_get_joint_num_dof.argtypes = [vp, C.c_char_p]
    L.cassie_sim_get_joint_num_dof.restype = ci
    L.cassie_sim_set_body_name_mass.argtypes = [vp, C.c_char_p, C.c_double]
    L.cassie_sim_set_body_name_mass.restype = None
    L.cassie_sim_get_body_name_mass.argtypes = [vp, C.c_char_p]
    L.cassie_sim_get_body_name_mass.restype = C.c_double
    for n in ('cassie_sim_set_const', 'cassie_sim_just_set_const'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = None
    for n in ('cassie_sim_foot_forces', 'cassie_sim_foot_positions', 'cassie_sim_foot_velocities', 'cassie_sim_cm_position', 'cassie_sim_cm_velocity',
              'cassie_sim_angular_momentum'):
        getattr(L, n).argtypes = [vp, cd]
        getattr(L, n).restype = None
    L.cassie_sim_heeltoe_forces.argtypes = [vp, cd, cd]
    L.cassie_sim_heeltoe_forces.restype = None
    for n in ('cassie_sim_check_obstacle_collision', 'cassie_sim_check_self_collision'):
        getattr(L, n).argtypes = [vp]
        getattr(L, n).restype = C.c_bool
    L.cassie_sim_geom_collision.argtypes = [vp, ci]
    L.cassie_sim_geom_collision.restype = C.c_bool
    _lib = L
    return L


def model_path(name='cassie'):
    """compiled model table shipped with the package (used where the reference's MJCF checkout is absent)."""
    return os.path.join(MODEL_DIR, name + '.cmodel')


def pd_rows(n, torque=None, pTarget=None, dTarget=None, pGain=None, dGain=None):
    """[n][52] compact motor-PD rows from 10-vectors (broadcast over envs) or [n][10] arrays."""
    rows = np.zeros((n, PD_WIDTH))
    for k, v in enumerate((torque, pTarget, dTarget, pGain, dGain)):
        if v is not None:
            rows[:, 10 * k:10 * k + 10] = np.asarray(v, dtype=np.float64)
    return rows


def _last_error():
    return lib().cassie_b200_last_error().decode()


class CassieBatch:
    """n_env independent Cassie simulators advanced in lock-step on one GPU."""

    def __init__(self, n_env, modelfile=None, device=0, precision=FP32):
        self.L = lib()
        self.n = int(n_env)
        path = modelfile or model_path()
        self.h = self.L.cassie_batch_init(path.encode(), self.n, int(device), int(precision))
        if not self.h:
            raise RuntimeError('cassie_batch_init failed: ' + _last_error())
        self.nq, self.nv = self.L.cassie_batch_nq(self.h), self.L.cassie_batch_nv(self.h)
        self.precision = precision
        self.device = int(device)

    def close(self):
        if getattr(self, 'h', None):
            self.L.cassie_batch_free(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @staticmethod
    def _dp(a):
        return a.ctypes.data_as(C.POINTER(C.c_double))

    # ---- stepping
    def set_pd(self, rows):
        rows = np.ascontiguousarray(rows, dtype=np.float64)
        assert rows.shape == (self.n, PD_WIDTH)
        self.L.cassie_batch_set_pd(self.h, self._dp(rows))

    def set_task_pd(self, rows):
        """taskPd rows [n, 60] (per leg torque, pTarget, dTarget, pGain, dGain [6]) or None to switch the branch off."""
        if rows is None:
            rc = self.L.cassie_batch_set_task_pd(self.h, None)
        else:
            a = np.ascontiguousarray(rows, dtype=np.float64).reshape(self.n, 60)
            rc = self.L.cassie_batch_set_task_pd(self.h, self._dp(a))
        if rc != 0:
            raise RuntimeError(_last_error())

    def set_pd_gait(self, amp=None, freq=None, phase=None):
        """open-loop gait on the motor-PD targets: pTarget_i(t) = row pTarget_i + amp[e, i] sin(2 pi freq[e] t + phase[e, i]), evaluated inside the kernel
        every control tick (t = ticks since reset / since this call x 0.5 ms); amp=None switches it off."""
        if amp is None:
            rc = self.L.cassie_batch_set_pd_gait(self.h, None, None, None)
        else:
            a = np.ascontiguousarray(np.broadcast_to(amp, (self.n, 10)), dtype=np.float64)
            f = np.ascontiguousarray(np.broadcast_to(freq, (self.n,)), dtype=np.float64)
            p = np.ascontiguousarray(np.broadcast_to(phase, (self.n, 10)), dtype=np.float64)
            rc = self.L.cassie_batch_set_pd_gait(self.h, self._dp(a), self._dp(f), self._dp(p))
        if rc != 0:
            raise RuntimeError(_last_error())

    def step(self, nticks=1):
        self.L.cassie_batch_step(self.h, int(nticks))

    def sync(self):
        self.L.cassie_batch_sync(self.h)

    def step_pd(self, pd_in_array, want_state=True):
        """AoS compatibility path: (pd_in_t * n) in, (state_out_t * n) out (cassie_sim_step_pd_batch)."""
        out = (state_out_t * self.n)() if want_state else None
        self.L.cassie_sim_step_pd_batch(self.h, C.byref(pd_in_array), C.byref(out) if want_state else None)
        return out

    def reset(self, mask=None):
        if mask is None:
            self.L.cassie_batch_reset(self.h, None)
        else:
            m = np.ascontiguousarray(mask, dtype=np.uint8)
            self.L.cassie_batch_reset(self.h, m.ctypes.data_as(C.c_void_p))

    def forward(self):
        self.L.cassie_batch_forward(self.h)

    def integrate_pos(self):
        self.L.cassie_batch_integrate_pos(self.h)

    # ---- state
    def _get(self, fn, w):
        out = np.zeros((self.n, w))
        fn(self.h, self._dp(out))
        return out

    def qpos(self):
        return self._get(self.L.cassie_batch_get_qpos, self.nq)

    def qvel(self):
        return self._get(self.L.cassie_batch_get_qvel, self.nv)

    def time(self):
        return self._get(self.L.cassie_batch_get_time, 1)[:, 0]

    def obs(self):
        return self._get(self.L.cassie_batch_get_obs, OBS_WIDTH)

    # ---- the estimator's host-side part for step_pd(): toe / heel forces, and the filters behind pelvis.position / translationalVelocity /
    # externalForce and terrain.height (one filter per environment, advanced once per step_pd call as the reference's 2 kHz estimator is)
    def enable_estimator(self, forces=True, filters=True):
        """HOST-side checker of the estimator (one filter object per environment, advanced per step_pd call); the product path is the
        in-kernel estimator (enable_estimator_device), which step_pd switches on by itself"""
        self.L.cassie_batch_enable_estimator_forces(self.h, 1 if (forces or filters) else 0)
        self.L.cassie_batch_enable_estimator_filter(self.h, 1 if filters else 0)

    def enable_estimator_device(self, on=True):
        """the estimator inside the step kernel: columns 96..111 of obs() / estimator() follow every tick of every launch; step_pd switches it
        on by itself at its first call, enable_estimator_device(False) keeps it off"""
        if self.L.cassie_batch_enable_estimator_device(self.h, 1 if on else 0) != 0:
            raise RuntimeError(_last_error())

    def estimator(self):
        """[n, 16]: position 3, translationalVelocity 3, externalForce 3, terrain.height, toeForce L 3, R 3"""
        out = np.zeros((self.n, EST_WIDTH))
        if self.L.cassie_batch_get_estimator(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    def reset_estimator(self, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self.L.cassie_batch_reset_estimator(self.h, None if m is None else m.ctypes.data)

    # ---- derived quantities (reference: the read-only queries of example/cassiemujoco.py:214-306, 815-819), one row per environment
    def enable_aux(self, on=True):
        if self.L.cassie_batch_enable_aux(self.h, 1 if on else 0) != 0:
            raise RuntimeError(_last_error())

    def aux(self):
        """[n, AUX_WIDTH] rows; slices are named in AUX (e.g. rows[:, AUX['foot_force']])."""
        out = np.zeros((self.n, AUX_WIDTH))
        if self.L.cassie_batch_get_aux(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    # ---- per-environment model constants (domain randomisation; reference: example/cassiemujoco.py:517-610 on one env)
    def _model_width(self, what):
        nb, ng = self.L.cassie_batch_nbody(self.h), self.L.cassie_batch_ngeom(self.h)
        return dict(body_mass=nb, body_ipos=3 * nb, dof_damping=self.nv, geom_friction=3 * ng)[what]

    def set_model(self, what, rows):
        """what in body_mass [n, nbody], body_ipos [n, 3 nbody], dof_damping [n, nv], geom_friction [n, 3 ngeom] (reference numbering)."""
        a = np.ascontiguousarray(rows, dtype=np.float64).reshape(self.n, self._model_width(what))
        if getattr(self.L, 'cassie_batch_set_' + what)(self.h, self._dp(a)) != 0:
            raise RuntimeError(_last_error())

    def get_model(self, what):
        out = np.zeros((self.n, self._model_width(what)))
        if getattr(self.L, 'cassie_batch_get_' + what)(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    def set_const(self, mask=None, reset_state=False):
        """mj_setConst on the device for the masked environments (all if None); reset_state=True adds cassie_sim_set_const's state reset."""
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        if self.L.cassie_batch_set_const(self.h, None if m is None else m.ctypes.data_as(C.c_void_p), 1 if reset_state else 0) != 0:
            raise RuntimeError(_last_error())

    # ---- placement of static geoms (stairs, floor tilt; reference: src/cassiemujoco.c:1466-1541, example/test_terrain.c:118-157)
    def set_geom_pose(self, name, pos=None, quat=None, size=None):
        """one placement shared by every environment: pos [3] / quat [4] in the geom's body frame, size [3]; None leaves that part alone.  As in
        MuJoCo a new size leaves the bounding radius alone.  Per-environment rows, if any, take this placement for the geom."""
        a = [None if v is None else np.ascontiguousarray(v, dtype=np.float64).reshape(w) for v, w in ((pos, 3), (quat, 4), (size, 3))]
        if self.L.cassie_batch_set_geom_pose(self.h, name.encode(), *[None if v is None else self._dp(v) for v in a]) != 0:
            raise RuntimeError(_last_error())

    def set_env_geom_pose(self, name, pos=None, quat=None, size=None, mask=None):
        """per-environment placement of a static plane / box: pos [3] or [n, 3], quat [4] or [n, 4], size [3] or [n, 3] (broadcast over the
        environments; None leaves that part alone); mask [n]: only the selected environments change.  A box's bounding radius follows |size|."""
        a = [None if v is None else np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (self.n, w))) for v, w in ((pos, 3), (quat, 4), (size, 3))]
        m = None if mask is None else np.ascontiguousarray(np.broadcast_to(np.asarray(mask, dtype=np.uint8), (self.n,)))
        if self.L.cassie_batch_set_env_geom_pose(self.h, name.encode(), *[None if v is None else self._dp(v) for v in a],
                                                 None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_geom_pose(self, name):
        """(pos [n, 3], quat [n, 4], size [n, 3]): the placement of a static plane / box each environment sees"""
        pos, quat, size = np.zeros((self.n, 3)), np.zeros((self.n, 4)), np.zeros((self.n, 3))
        if self.L.cassie_batch_get_env_geom_pose(self.h, name.encode(), self._dp(pos), self._dp(quat), self._dp(size)) != 0:
            raise RuntimeError(_last_error())
        return pos, quat, size

    def clear_env_geom_poses(self):
        """drop the per-environment placements: every environment follows the shared placement again"""
        if self.L.cassie_batch_clear_env_geom_poses(self.h) != 0:
            raise RuntimeError(_last_error())

    # ---- per-environment terrain (terrain curricula: promote / demote environments between terrain types and difficulty levels at their resets)
    def set_env_hfield(self, terrain=None, pos=None, size=None, mask=None):
        """which bank entry each environment stands on and where and how large its height field is: terrain [n] (or one int) in [0, K) of
        set_hfield_data, pos [3] or [n, 3] (in the height field's body frame; it stays axis-aligned), size [4] or [n, 4] (x half-extent, y half-extent,
        elevation scale, base thickness); None leaves that part alone; mask [n]: only the selected environments change.  A bad value raises and
        changes nothing.  Reset and snapshot restore leave these alone."""
        t = None if terrain is None else np.ascontiguousarray(np.broadcast_to(np.asarray(terrain, dtype=np.int32), (self.n,)))
        a = [None if v is None else np.ascontiguousarray(np.broadcast_to(np.asarray(v, dtype=np.float64), (self.n, w))) for v, w in ((pos, 3), (size, 4))]
        m = None if mask is None else np.ascontiguousarray(np.broadcast_to(np.asarray(mask, dtype=np.uint8), (self.n,)))
        if self.L.cassie_batch_set_env_hfield(self.h, None if t is None else t.ctypes.data_as(C.POINTER(C.c_int)), *[None if v is None else self._dp(v) for v in a],
                                              None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_hfield(self):
        """(terrain [n] int32, pos [n, 3], size [n, 4]): the bank entry, height-field position and size each environment sees"""
        t, pos, size = np.zeros(self.n, dtype=np.int32), np.zeros((self.n, 3)), np.zeros((self.n, 4))
        if self.L.cassie_batch_get_env_hfield(self.h, t.ctypes.data_as(C.POINTER(C.c_int)), self._dp(pos), self._dp(size)) != 0:
            raise RuntimeError(_last_error())
        return t, pos, size

    def clear_env_hfield(self):
        """back to terrain e % K and the shared position and size"""
        if self.L.cassie_batch_clear_env_hfield(self.h) != 0:
            raise RuntimeError(_last_error())

    # ---- per-environment body offsets (where a load or tray sits, link and mounting offsets: domain randomisation)
    def set_env_body_pos(self, pos, mask=None):
        """each environment's MuJoCo body_pos: pos [nbody, 3] (all environments) or [n, nbody, 3], in model body order; mask [n]: only the selected
        environments change.  The world body, bodies welded to the world and the extra free body keep the model's offsets (a change raises, and nothing
        changes).  The mj_setConst constants are not refreshed by this: call set_const, as with the reference.  Reset and snapshot restore leave the
        offsets alone."""
        nb = self.L.cassie_batch_nbody(self.h)
        a = np.ascontiguousarray(np.broadcast_to(np.asarray(pos, dtype=np.float64), (self.n, nb, 3)))
        m = None if mask is None else np.ascontiguousarray(np.broadcast_to(np.asarray(mask, dtype=np.uint8), (self.n,)))
        if self.L.cassie_batch_set_env_body_pos(self.h, self._dp(a), None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_body_pos(self):
        """[n, nbody, 3]: the body offsets each environment sees (the model's without rows)"""
        out = np.zeros((self.n, self.L.cassie_batch_nbody(self.h), 3))
        if self.L.cassie_batch_get_env_body_pos(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    def clear_env_body_pos(self):
        """back to the model's body offsets and the kernel instances that ran before"""
        if self.L.cassie_batch_clear_env_body_pos(self.h) != 0:
            raise RuntimeError(_last_error())

    # ---- per-environment actuators (actuator latency and torque saturation: sim-to-real randomisation) and the controller-stage state
    def _act_lib(self):
        L = self.L
        if not getattr(L, '_act_bound', False):
            vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
            L.cassie_batch_set_env_actuators.argtypes = [vp, dp, dp, ip, vp]
            L.cassie_batch_get_env_actuators.argtypes = [vp, dp, dp, ip]
            L.cassie_batch_clear_env_actuators.argtypes = [vp]
            L.cassie_batch_get_actuator_state.argtypes = [vp, dp, ip, dp, dp]
            L.cassie_batch_set_actuator_state.argtypes = [vp, dp, ip, dp, dp, vp]
            for n in ('set_env_actuators', 'get_env_actuators', 'clear_env_actuators', 'get_actuator_state', 'set_actuator_state'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._act_bound = True
        return L

    @staticmethod
    def _arr(a, dtype, shape):
        return None if a is None else np.ascontiguousarray(np.broadcast_to(np.asarray(a, dtype=dtype), shape))

    def set_env_actuators(self, ctrlrange=None, rpm=None, delay=None, mask=None):
        """each environment's actuators, per motor (10, in the model's actuator order): ctrlrange [nu, 2] or [n, nu, 2] -- MuJoCo's actuator_ctrlrange
        (lo, hi): the clamp of ctrl and motor()'s peak torque --, rpm [nu] or [n, nu] -- the no-load speed (actuator_user) --, delay [nu] or [n, nu] --
        the torque delay in control ticks, 0..6 (6: the reference's).  A part left None is kept; mask [n]: only the selected environments change.  A
        non-finite value, lo >= hi, rpm <= 0 or a delay outside 0..6 raises, and nothing changes.  Reset and snapshot restore leave the rows alone."""
        L, nu = self._act_lib(), NU
        cr = self._arr(ctrlrange, np.float64, (self.n, nu, 2))
        rp = self._arr(rpm, np.float64, (self.n, nu))
        m = self._arr(mask, np.uint8, (self.n,))
        dl = None
        if delay is not None:   # checked before the conversion to int32, which would wrap a large value into the range
            d = np.broadcast_to(np.asarray(delay, dtype=np.float64), (self.n, nu))
            dm = d if m is None else d[m != 0]
            if not np.all(np.isfinite(dm)) or np.any(dm != np.round(dm)) or np.any((dm < 0) | (dm > LINE_MAX)):
                raise RuntimeError('set_env_actuators: delay must be whole ticks in 0..%d' % LINE_MAX)
            dl = np.ascontiguousarray(np.where(np.isfinite(d) & (d >= 0) & (d <= LINE_MAX), d, 0).astype(np.int32))   # unmasked rows are not read
        ptr = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
        if L.cassie_batch_set_env_actuators(self.h, ptr(cr, C.c_double), ptr(rp, C.c_double), ptr(dl, C.c_int), None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_actuators(self):
        """(ctrlrange [n, nu, 2], rpm [n, nu], delay [n, nu] int): the actuators each environment sees (the model's without rows)"""
        L, nu = self._act_lib(), NU
        cr, rp, dl = np.zeros((self.n, nu, 2)), np.zeros((self.n, nu)), np.zeros((self.n, nu), dtype=np.int32)
        if L.cassie_batch_get_env_actuators(self.h, self._dp(cr), self._dp(rp), dl.ctypes.data_as(C.POINTER(C.c_int))) != 0:
            raise RuntimeError(_last_error())
        return cr, rp, dl

    def clear_env_actuators(self):
        """back to the model's actuators and the kernel instances that ran before"""
        if self._act_lib().cassie_batch_clear_env_actuators(self.h) != 0:
            raise RuntimeError(_last_error())

    # ---- per-environment mechanics (link inertia, rotor armature, leaf springs: sim-to-real randomisation)
    def _mech_lib(self):
        L = self.L
        if not getattr(L, '_mech_bound', False):
            vp, dp = C.c_void_p, C.POINTER(C.c_double)
            L.cassie_batch_set_env_mechanics.argtypes = [vp, dp, dp, dp, dp, vp]
            L.cassie_batch_get_env_mechanics.argtypes = [vp, dp, dp, dp, dp]
            L.cassie_batch_clear_env_mechanics.argtypes = [vp]
            L.cassie_batch_njnt.argtypes = [vp]
            for n in ('set_env_mechanics', 'get_env_mechanics', 'clear_env_mechanics', 'njnt'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._mech_bound = True
        return L

    def _mech_shapes(self):
        L = self._mech_lib()
        return (L.cassie_batch_nbody(self.h), 3), (self.nv,), (L.cassie_batch_njnt(self.h),), (L.cassie_batch_njnt(self.h),)

    def set_env_mechanics(self, inertia=None, armature=None, stiffness=None, springref=None, mask=None):
        """each environment's mechanics: inertia [nbody, 3] or [n, nbody, 3] -- MuJoCo's body_inertia, the principal moments, in model body order --,
        armature [nv] or [n, nv] -- dof_armature --, stiffness and springref [njnt] or [n, njnt] -- jnt_stiffness and qpos_spring of every hinge (slide,
        ball and free joints must keep what env_mechanics() reports).  A part left None is kept; mask [n]: only the selected environments change.  A
        non-finite value, a negative moment / armature / stiffness, moments with A + B < C, or a change to the world body, a body welded to the world or
        the extra free body raises, and nothing changes.  As in MuJoCo the mj_setConst constants are not refreshed: call set_const.  Reset and snapshot
        restore leave the rows alone."""
        L = self._mech_lib()
        a = [self._arr(v, np.float64, (self.n,) + sh) for v, sh in zip((inertia, armature, stiffness, springref), self._mech_shapes())]
        m = self._arr(mask, np.uint8, (self.n,))
        if L.cassie_batch_set_env_mechanics(self.h, *[None if v is None else self._dp(v) for v in a], None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_mechanics(self):
        """dict of inertia [n, nbody, 3], armature [n, nv], stiffness [n, njnt], springref [n, njnt]: what each environment sees (the model's without rows)"""
        L = self._mech_lib()
        out = [np.zeros((self.n,) + sh) for sh in self._mech_shapes()]
        if L.cassie_batch_get_env_mechanics(self.h, *[self._dp(v) for v in out]) != 0:
            raise RuntimeError(_last_error())
        return dict(zip(('inertia', 'armature', 'stiffness', 'springref'), out))

    def clear_env_mechanics(self):
        """back to the model's inertias, armatures and springs and the kernel instances that ran before"""
        if self._mech_lib().cassie_batch_clear_env_mechanics(self.h) != 0:
            raise RuntimeError(_last_error())

    # ---- per-environment contact softness (ground stiffness, damping and impedance: sim-to-real randomisation)
    def _contact_lib(self):
        L = self.L
        if not getattr(L, '_contact_bound', False):
            vp, dp = C.c_void_p, C.POINTER(C.c_double)
            L.cassie_batch_set_env_contact.argtypes = [vp, dp, dp, dp, vp]
            L.cassie_batch_get_env_contact.argtypes = [vp, dp, dp, dp]
            L.cassie_batch_clear_env_contact.argtypes = [vp]
            for n in ('set_env_contact', 'get_env_contact', 'clear_env_contact'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._contact_bound = True
        return L

    def _contact_shapes(self):
        ng = self.L.cassie_batch_ngeom(self.h)
        return (ng, 2), (ng, 5), (ng,)

    def set_env_contact(self, solref=None, solimp=None, solmix=None, mask=None):
        """each environment's contact softness, per geom (model geom order): solref [ngeom, 2] or [n, ngeom, 2] -- MuJoCo's geom_solref, (timeconst,
        dampratio) or direct (-stiffness, -damping) --, solimp [ngeom, 5] or [n, ngeom, 5] -- geom_solimp (dmin, dmax, width, midpoint, power) --, solmix
        [ngeom] or [n, ngeom] -- geom_solmix.  Each contact mixes its two geoms' values as MuJoCo's mj_contactParam does.  A part left None is kept; mask
        [n]: only the selected environments change.  A non-finite value, a solref with mixed signs, a solimp outside 0 < dmin, dmax, midpoint < 1,
        width >= 0, power >= 1, or a negative solmix raises, and nothing changes.  Entries of geoms that never collide are ignored.  Reset and snapshot
        restore leave the rows alone."""
        L = self._contact_lib()
        a = [self._arr(v, np.float64, (self.n,) + sh) for v, sh in zip((solref, solimp, solmix), self._contact_shapes())]
        m = self._arr(mask, np.uint8, (self.n,))
        if L.cassie_batch_set_env_contact(self.h, *[None if v is None else self._dp(v) for v in a], None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_contact(self):
        """dict of solref [n, ngeom, 2], solimp [n, ngeom, 5], solmix [n, ngeom]: what each environment sees (the model's without rows)"""
        L = self._contact_lib()
        out = [np.zeros((self.n,) + sh) for sh in self._contact_shapes()]
        if L.cassie_batch_get_env_contact(self.h, *[self._dp(v) for v in out]) != 0:
            raise RuntimeError(_last_error())
        return dict(zip(('solref', 'solimp', 'solmix'), out))

    def clear_env_contact(self):
        """back to the model's contact softness and the kernel instances that ran before"""
        if self._contact_lib().cassie_batch_clear_env_contact(self.h) != 0:
            raise RuntimeError(_last_error())

    # ---- per-environment applied forces (perturbation: pushes on any body, joint-space disturbance torques; state, as in mjData)
    def _applied_lib(self):
        L = self.L
        if not getattr(L, '_applied_bound', False):
            vp, dp = C.c_void_p, C.POINTER(C.c_double)
            L.cassie_batch_set_applied_forces.argtypes = [vp, dp, dp, vp]
            L.cassie_batch_get_applied_forces.argtypes = [vp, dp, dp]
            L.cassie_batch_enable_applied_forces.argtypes = [vp, C.c_int]
            for n in ('set_applied_forces', 'get_applied_forces', 'enable_applied_forces'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._applied_bound = True
        return L

    def _applied_shapes(self):
        return (self.L.cassie_batch_nbody(self.h), 6), (self.nv,)

    def set_applied_forces(self, xfrc=None, qfrc=None, mask=None):
        """each environment's applied forces: xfrc [nbody, 6] or [n, nbody, 6] -- MuJoCo's xfrc_applied, force xyz and torque xyz in the world frame at the
        body's centre of mass, model body order --, qfrc [nv] or [n, nv] -- qfrc_applied, the extra free body's dofs included.  A part left None is kept;
        mask [n]: only the selected environments change.  A non-finite value raises, and nothing changes.  State: reset() zeroes both, clear_forces() the
        body wrenches; snapshots carry them.  apply_force's slot adds to the rows."""
        L = self._applied_lib()
        a = [self._arr(v, np.float64, (self.n,) + sh) for v, sh in zip((xfrc, qfrc), self._applied_shapes())]
        m = self._arr(mask, np.uint8, (self.n,))
        if L.cassie_batch_set_applied_forces(self.h, *[None if v is None else self._dp(v) for v in a], None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def applied_forces(self):
        """dict of xfrc [n, nbody, 6], qfrc [n, nv]: what the rows hold (zeros without rows)"""
        L = self._applied_lib()
        out = [np.zeros((self.n,) + sh) for sh in self._applied_shapes()]
        if L.cassie_batch_get_applied_forces(self.h, *[self._dp(v) for v in out]) != 0:
            raise RuntimeError(_last_error())
        return dict(zip(('xfrc', 'qfrc'), out))

    def enable_applied_forces(self, on=True):
        """on: zeroed rows, for writing through torch_view('applied') only; off: drop the rows and their forces, back to the kernel instances that ran before"""
        if self._applied_lib().cassie_batch_enable_applied_forces(self.h, 1 if on else 0) != 0:
            raise RuntimeError(_last_error())

    # ---- sensor models drawn in the step kernel (encoder offsets and noise, IMU mount, bias and noise: sim-to-real randomisation)
    def _sensor_lib(self):
        L = self.L
        if not getattr(L, '_sensor_bound', False):
            vp, dp, up = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_ulonglong)
            L.cassie_batch_set_env_sensors.argtypes = [vp, dp, dp, dp, dp, dp, vp]
            L.cassie_batch_get_env_sensors.argtypes = [vp, dp, dp, dp, dp, dp]
            L.cassie_batch_clear_env_sensors.argtypes = [vp]
            L.cassie_batch_seed_sensors.argtypes = [vp, C.c_ulonglong, vp]
            L.cassie_batch_get_sensor_rng.argtypes = [vp, up, up]
            for n in ('set_env_sensors', 'get_env_sensors', 'clear_env_sensors', 'seed_sensors', 'get_sensor_rng'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._sensor_bound = True
        return L

    _SENSOR_SHAPES = (('enc_offset', (16,)), ('enc_noise', (16,)), ('imu_quat', (4,)), ('imu_bias', (6,)), ('imu_noise', (9,)))

    def set_env_sensors(self, enc_offset=None, enc_noise=None, imu_quat=None, imu_bias=None, imu_noise=None, mask=None):
        """each environment's sensor model, applied every tick to what the controller, the safety layer, the encoder filters and the estimator measure:
        enc_offset / enc_noise [16] or [n, 16] -- offset and noise std of the encoders in cassie_out order (10 drives, 6 joints), output radians --,
        imu_quat [4] or [n, 4] -- the IMU mount q_m (w x y z, normalised on write): orientation q (x) q_m, rates and accelerations R_m' v --, imu_bias [6]
        or [n, 6] -- gyro, accelerometer --, imu_noise [9] or [n, 9] -- std of the orientation (rad), gyro, accelerometer.  A part left None is kept;
        mask [n]: only the selected environments change.  A non-finite value, a negative std or a zero quaternion raises, and nothing changes.  Reset and
        snapshot restore leave the rows alone.  The first call seeds the generator as seed_sensors(0)."""
        L = self._sensor_lib()
        a = [self._arr(v, np.float64, (self.n,) + sh) for v, (_, sh) in zip((enc_offset, enc_noise, imu_quat, imu_bias, imu_noise), self._SENSOR_SHAPES)]
        m = self._arr(mask, np.uint8, (self.n,))
        if L.cassie_batch_set_env_sensors(self.h, *[None if v is None else self._dp(v) for v in a], None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_sensors(self):
        """dict of enc_offset [n, 16], enc_noise [n, 16], imu_quat [n, 4], imu_bias [n, 6], imu_noise [n, 9]: what the rows hold (the zero model without rows)"""
        L = self._sensor_lib()
        out = [np.zeros((self.n,) + sh) for _, sh in self._SENSOR_SHAPES]
        if L.cassie_batch_get_env_sensors(self.h, *[self._dp(v) for v in out]) != 0:
            raise RuntimeError(_last_error())
        return dict(zip([k for k, _ in self._SENSOR_SHAPES], out))

    def clear_env_sensors(self):
        """back to perfect sensors and the kernel instances that ran before"""
        if self._sensor_lib().cassie_batch_clear_env_sensors(self.h) != 0:
            raise RuntimeError(_last_error())

    def seed_sensors(self, seed, mask=None):
        """environment i draws from key seed + i, counter 0 (mask [n]: only the selected environments); set_env_sensors first"""
        m = self._arr(mask, np.uint8, (self.n,))
        if self._sensor_lib().cassie_batch_seed_sensors(self.h, C.c_ulonglong(int(seed) & (2 ** 64 - 1)), None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def sensor_rng(self):
        """(key [n], counter [n]) uint64: the generator each environment draws from; step launches advance the counter by their tick count"""
        key, ctr = np.zeros(self.n, dtype=np.uint64), np.zeros(self.n, dtype=np.uint64)
        up = C.POINTER(C.c_ulonglong)
        if self._sensor_lib().cassie_batch_get_sensor_rng(self.h, key.ctypes.data_as(up), ctr.ctypes.data_as(up)) != 0:
            raise RuntimeError(_last_error())
        return key, ctr

    # ---- per-tick traces of multi-tick launches
    def _trace_lib(self):
        L = self.L
        if not getattr(L, '_trace_bound', False):
            vp, ip = C.c_void_p, C.POINTER(C.c_int)
            L.cassie_batch_set_trace.argtypes = [vp, ip, ip, C.c_int, C.c_int]
            L.cassie_batch_trace_ticks.argtypes = [vp]
            L.cassie_batch_get_trace.argtypes = [vp, C.POINTER(C.c_double)]
            for n in ('set_trace', 'trace_ticks', 'get_trace'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._trace_bound = True
        return L

    def set_trace(self, columns, max_ticks=50):
        """trace k <= TRACE_MAX columns at every tick of a step launch: columns is a list of (source, column) pairs, source one of TRACE_QPOS,
        TRACE_QVEL, TRACE_OBS, TRACE_AUX (enable_aux first), TRACE_FRAME (set_frames first); max_ticks slots T per environment, the last T ticks of a
        longer launch kept in order.  An empty list drops the trace.  A bad column raises, and nothing changes.  See include/cassie_b200.h."""
        cols = [(int(s), int(c)) for s, c in columns]
        src = (C.c_int * max(1, len(cols)))(*[s for s, _ in cols])
        col = (C.c_int * max(1, len(cols)))(*[c for _, c in cols])
        if self._trace_lib().cassie_batch_set_trace(self.h, src, col, len(cols), int(max_ticks)) != 0:
            raise RuntimeError(_last_error())
        self._trace_shape = (int(max_ticks), len(cols)) if cols else None

    def trace_ticks(self):
        """slots the last step launch wrote: min(nticks, max_ticks)"""
        return int(self._trace_lib().cassie_batch_trace_ticks(self.h))

    def trace(self):
        """the slots the last step launch wrote, [n, trace_ticks(), k] (a synchronous copy)"""
        shape = getattr(self, '_trace_shape', None)
        if shape is None:
            raise RuntimeError('no trace is set (set_trace)')
        out = np.zeros((self.n,) + shape)
        if self._trace_lib().cassie_batch_get_trace(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out[:, :self.trace_ticks()]

    # ---- contact lists of step and forward launches
    def _contacts_lib(self):
        L = self.L
        if not getattr(L, '_contacts_bound', False):
            vp = C.c_void_p
            L.cassie_batch_enable_contacts.argtypes = [vp, C.c_int]
            L.cassie_batch_get_contacts.argtypes = [vp, C.POINTER(C.c_double)]
            L.cassie_batch_name2id.argtypes = [vp, C.c_char_p, C.c_char_p]
            L.cassie_batch_id2name.argtypes = [vp, C.c_char_p, C.c_int]
            L.cassie_batch_id2name.restype = C.c_char_p
            for n in ('enable_contacts', 'get_contacts', 'name2id'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._contacts_bound = True
        return L

    def enable_contacts(self, on=True):
        """contact-list rows: every step and forward launch then lists the contacts of its last sub-step (contacts()); on=False frees them and the
        batch runs the instance it ran before.  A batch with a per-tick trace refuses them.  See include/cassie_b200.h."""
        if self._contacts_lib().cassie_batch_enable_contacts(self.h, 1 if on else 0) != 0:
            raise RuntimeError(_last_error())

    def contacts(self):
        """dict of the contact lists (a synchronous copy): count, found, dropped [n]; geom [n, 12, 2] int (model geom ids, -1 in unused slots); dim,
        dist, mu [n, 12]; pos [n, 12, 3]; frame [n, 12, 3, 3] (row 0 the normal from geom1 to geom2); force [n, 12, 6] (mj_contactForce, contact
        frame); world_force [n, 12, 3] = frame' force[:3], the force on geom2 in the world frame; efc [n, 12] int (first constraint row)"""
        rows = np.zeros((self.n, CON_WIDTH))
        if self._contacts_lib().cassie_batch_get_contacts(self.h, self._dp(rows)) != 0:
            raise RuntimeError(_last_error())
        s = rows[:, CON_HEAD:].reshape(self.n, CON_MAX, CON_SLOT)
        frame = s[:, :, CON['frame']].reshape(self.n, CON_MAX, 3, 3)
        force = s[:, :, CON['force']].copy()
        return dict(count=rows[:, 0].astype(int), found=rows[:, 1].astype(int), dropped=rows[:, 2].astype(int),
                    geom=s[:, :, 0:2].astype(int), dim=s[:, :, CON['dim']].astype(int), dist=s[:, :, CON['dist']].copy(), mu=s[:, :, CON['mu']].copy(),
                    efc=s[:, :, CON['efc']].astype(int), pos=s[:, :, CON['pos']].copy(), frame=frame.copy(), force=force,
                    world_force=np.einsum('ecji,ecj->eci', frame, force[:, :, :3]))

    def name2id(self, kind, name):
        """id of a named body ('body' / 'xbody'), joint, geom, site or camera of the compiled model, or -1: an unknown name, or a kind the compiled
        model keeps no names of (mj_name2id)"""
        return int(self._contacts_lib().cassie_batch_name2id(self.h, kind.encode(), name.encode()))

    def id2name(self, kind, i):
        """name of object i of a kind name2id resolves, or None: out of range, unnamed, or a kind without names (mj_id2name)"""
        r = self._contacts_lib().cassie_batch_id2name(self.h, kind.encode(), int(i))
        return None if r is None else r.decode()

    def actuator_state(self):
        """dict of the controller-stage state: torque_delay [n, 10, 6] (slot 0 newest), drive_filter [n, 10, 9] int32, joint_x [n, 6, 4], joint_y [n, 6, 3]"""
        L = self._act_lib()
        td, df, jx, jy = np.zeros((self.n, 10, 6)), np.zeros((self.n, 10, 9), dtype=np.int32), np.zeros((self.n, 6, 4)), np.zeros((self.n, 6, 3))
        if L.cassie_batch_get_actuator_state(self.h, self._dp(td), df.ctypes.data_as(C.POINTER(C.c_int)), self._dp(jx), self._dp(jy)) != 0:
            raise RuntimeError(_last_error())
        return dict(torque_delay=td, drive_filter=df, joint_x=jx, joint_y=jy)

    def set_actuator_state(self, torque_delay=None, drive_filter=None, joint_x=None, joint_y=None, mask=None):
        """writes the parts given (shapes as actuator_state(), or one environment's broadcast to all); mask [n]: only the selected environments change"""
        L = self._act_lib()
        td = self._arr(torque_delay, np.float64, (self.n, 10, 6))
        df = self._arr(drive_filter, np.int32, (self.n, 10, 9))
        jx = self._arr(joint_x, np.float64, (self.n, 6, 4))
        jy = self._arr(joint_y, np.float64, (self.n, 6, 3))
        m = self._arr(mask, np.uint8, (self.n,))
        ptr = lambda a, t: None if a is None else a.ctypes.data_as(C.POINTER(t))
        if L.cassie_batch_set_actuator_state(self.h, ptr(td, C.c_double), ptr(df, C.c_int), ptr(jx, C.c_double), ptr(jy, C.c_double),
                                             None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def set_hfield_size(self, size):
        """the shared height-field size [4]; every environment's position and size go back to the shared ones, terrain selections stay"""
        a = np.ascontiguousarray(np.asarray(size, dtype=np.float64).reshape(4))
        if self.L.cassie_batch_set_hfield_size(self.h, self._dp(a)) != 0:
            raise RuntimeError(_last_error())

    def hfield_size(self):
        out = np.zeros(4)
        if self.L.cassie_batch_get_hfield_size(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    # ---- frames: named bodies / sites written by every step and forward (reference: xpos, xquat, get_site_xpos, get_site_quat, body_vel,
    # get_body_contact_force of example/cassiemujoco.py)
    def set_frames(self, names, kinds=None):
        """track `names` (bodies, or sites where kinds[i] == FRAME_SITE; kinds=None: all bodies); [] drops the rows.  From the next launch on,
        frames() holds per environment and frame the pose of the state the last physics sub-step started from and that sub-step's velocity and
        contact force, laid out as FRAME (pos, quat, vel, cfrc slices of FRAME_WIDTH)."""
        names = list(names)
        kinds = [FRAME_BODY] * len(names) if kinds is None else [int(k) for k in kinds]
        if len(kinds) != len(names):
            raise ValueError('one kind per frame name')
        arr = (C.c_char_p * max(1, len(names)))(*[n.encode() for n in names])
        ks = (C.c_int * max(1, len(kinds)))(*kinds)
        self.L.cassie_batch_set_frames.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.c_int]
        if self.L.cassie_batch_set_frames(self.h, arr, ks, len(names)) != 0:
            raise RuntimeError(_last_error())

    def nframes(self):
        self.L.cassie_batch_nframes.argtypes = [C.c_void_p]
        return int(self.L.cassie_batch_nframes(self.h))

    def frame_jacobian(self, i):
        """(jacp, jacr) [n, 3, nv] of frame i (its index in set_frames) at the CURRENT state, as the reference's get_jacobian_full(_site): one launch
        that writes nothing else"""
        jacp, jacr = np.zeros((self.n, 3, self.nv)), np.zeros((self.n, 3, self.nv))
        self.L.cassie_batch_frame_jacobian.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        if self.L.cassie_batch_frame_jacobian(self.h, int(i), self._dp(jacp), self._dp(jacr)) != 0:
            raise RuntimeError(_last_error())
        return jacp, jacr

    def frames(self):
        """[n, nframes, FRAME_WIDTH] rows of the frames set with set_frames"""
        out = np.zeros((self.n, self.nframes(), FRAME_WIDTH))
        self.L.cassie_batch_get_frames.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        if self.L.cassie_batch_get_frames(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    # ---- accelerations (reference: qacc, get_body_acceleration of example/cassiemujoco.py): by-products of every step and forward
    def enable_accelerations(self, on=True):
        """allocate (on) or drop the acceleration rows.  From the next step or forward on, qacc() holds the constraint-solved qacc of the last physics
        sub-step and body_accelerations() the cacc of every frame of set_frames (zeros for sites); set_frames reallocates the rows to its width"""
        self.L.cassie_batch_enable_accelerations.argtypes = [C.c_void_p, C.c_int]
        if self.L.cassie_batch_enable_accelerations(self.h, 1 if on else 0) != 0:
            raise RuntimeError(_last_error())

    def _accelerations(self, qacc, cacc):
        self.L.cassie_batch_get_accelerations.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        if self.L.cassie_batch_get_accelerations(self.h, self._dp(qacc) if qacc is not None else None, self._dp(cacc) if cacc is not None else None) != 0:
            raise RuntimeError(_last_error())

    def qacc(self):
        """[n, nv] qacc of the last step / forward (after a step: the value the warm start keeps, before the implicit-damping correction)"""
        out = np.zeros((self.n, self.nv))
        self._accelerations(out, None)
        return out

    def body_accelerations(self):
        """[n, nframes, 6] cacc of the frames (com-based [angular; linear], gravity included as cacc(world) = (0, 0, 0, -g); sites read zero)"""
        out = np.zeros((self.n, self.nframes(), 6))
        self._accelerations(None, out)
        return out

    # ---- dynamics at the current state (reference: full_mass_matrix, constraint_jacobian / constraint_error, centroid_inertia of
    # example/cassiemujoco.py): mass matrix, bias forces, connect-equality rows
    def compute_dynamics(self):
        """enqueue one dynamics launch on the batch's stream (asynchronous): M, bias, connect rows and the centre-of-mass offset of the CURRENT state
        into the device rows (torch_view('dyn')); nothing else is written"""
        self.L.cassie_batch_dynamics.argtypes = [C.c_void_p]
        if self.L.cassie_batch_dynamics(self.h) != 0:
            raise RuntimeError(_last_error())

    def neq(self):
        self.L.cassie_batch_neq.argtypes = [C.c_void_p]
        return int(self.L.cassie_batch_neq(self.h))

    def dynamics(self):
        """what the last compute_dynamics() wrote, as numpy arrays: M [n, nv, nv], bias [n, nv] (qfrc_bias), J_eq [n, 3 neq, nv] and eq_err [n, 3 neq]
        (the connect equalities' efc_J / efc_pos rows), Icm [n, 3, 3] (the reference's centroid_inertia formula)"""
        ne = 3 * self.neq()
        out = dict(M=np.zeros((self.n, self.nv, self.nv)), bias=np.zeros((self.n, self.nv)), J_eq=np.zeros((self.n, ne, self.nv)), eq_err=np.zeros((self.n, ne)),
                   Icm=np.zeros((self.n, 3, 3)))
        self.L.cassie_batch_get_dynamics.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * 5
        if self.L.cassie_batch_get_dynamics(self.h, *(self._dp(out[k]) for k in ('M', 'bias', 'J_eq', 'eq_err', 'Icm'))) != 0:
            raise RuntimeError(_last_error())
        return out

    # ---- inverse dynamics at the current state (MuJoCo 2.1.0's mj_inverse, continuous time): the generalised force that produces a given qacc, contact and
    # loop-closure forces included; applied forces and actuation are part of what it returns
    def compute_inverse(self, qacc=None):
        """enqueue one inverse launch on the batch's stream (asynchronous) at the CURRENT state: qacc [n, nv] (host) is uploaded first; None uses
        torch_view('inv_qacc') as the caller left it on the device (for example copied from torch_view('acc')[:, ACC['qacc']]), with no host
        synchronisation, copy or allocation after the first call.  The result goes to the device rows (torch_view('inv')); nothing else is written"""
        self.L.cassie_batch_inverse.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        a = None
        if qacc is not None:
            a = np.ascontiguousarray(np.asarray(qacc, dtype=np.float64).reshape(self.n, self.nv))
        if self.L.cassie_batch_inverse(self.h, self._dp(a) if a is not None else None) != 0:
            raise RuntimeError(_last_error())

    def inverse(self):
        """what the last compute_inverse() wrote, as numpy arrays: qfrc_inverse [n, nv] (M qacc + qfrc_bias - qfrc_passive - qfrc_constraint),
        qfrc_constraint [n, nv], and per environment nefc, ncon and dropped [n] (constraint rows, contacts with rows, contacts dropped at the capacities)"""
        out = dict(qfrc_inverse=np.zeros((self.n, self.nv)), qfrc_constraint=np.zeros((self.n, self.nv)))
        counts = np.zeros((self.n, 3), dtype=np.int32)
        self.L.cassie_batch_get_inverse.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_int)]
        if self.L.cassie_batch_get_inverse(self.h, self._dp(out['qfrc_inverse']), self._dp(out['qfrc_constraint']), counts.ctypes.data_as(C.POINTER(C.c_int))) != 0:
            raise RuntimeError(_last_error())
        out.update(nefc=counts[:, 0].copy(), ncon=counts[:, 1].copy(), dropped=counts[:, 2].copy())
        return out

    # ---- terrain rays (height scans; the reference's rangefinders, example/cassiemujoco.py sense_ground): cast against each environment's static
    # geoms (floor, height field, boxes, with its own placement and terrain) at the CURRENT state; the robot and the extra free body are not seen
    def set_rays(self, origin, direction, frame='heading', max_dist=3.0):
        """origin / direction [k, 3] (directions are normalised), frame 'heading' (root position and yaw, level), 'root' (root pose) or 'world' (or
        RAY_HEADING / RAY_ROOT / RAY_WORLD), or one kind per ray ([k] of those), max_dist scalar or [k]; k = 0 drops the table.  Reallocates the rows: a torch_view('rays') taken
        before it must not be used after it."""
        o = np.ascontiguousarray(np.asarray(origin, dtype=np.float64).reshape(-1, 3))
        k = len(o)
        d = np.ascontiguousarray(np.broadcast_to(np.asarray(direction, dtype=np.float64), (k, 3)))
        if isinstance(frame, (str, int, np.integer)):
            frame = [frame] * k
        f = [RAY_FRAMES[x] if isinstance(x, str) else int(x) for x in frame]
        if len(f) != k:
            raise ValueError('one frame kind per ray')
        fr = (C.c_int * max(1, k))(*f)
        m = np.ascontiguousarray(np.broadcast_to(np.asarray(max_dist, dtype=np.float64), (k,)))
        self.L.cassie_batch_set_rays.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_double), C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_int]
        if self.L.cassie_batch_set_rays(self.h, fr, self._dp(o), self._dp(d), self._dp(m), k) != 0:
            raise RuntimeError(_last_error())

    def set_height_scan(self, xs, ys, z_start=1.0, max_dist=3.0):
        """a height scan: the grid xs x ys (x slowest) in the heading frame, rays along -z from z_start above the root"""
        gx, gy = np.meshgrid(np.asarray(xs, dtype=np.float64), np.asarray(ys, dtype=np.float64), indexing='ij')
        org = np.stack([gx.ravel(), gy.ravel(), np.full(gx.size, float(z_start))], axis=1)
        self.set_rays(org, [0.0, 0.0, -1.0], 'heading', max_dist)

    def nrays(self):
        self.L.cassie_batch_nrays.argtypes = [C.c_void_p]
        return int(self.L.cassie_batch_nrays(self.h))

    def raycast(self):
        """enqueue one cast of every ray of every environment on the batch's stream (asynchronous), at the CURRENT state; nothing else is written"""
        self.L.cassie_batch_raycast.argtypes = [C.c_void_p]
        if self.L.cassie_batch_raycast(self.h) != 0:
            raise RuntimeError(_last_error())

    def rays(self):
        """[n, k, RAY_SLOT] rows of the last raycast(): distance (-1: none), world z of the hit (end point when none), static geom slot (-1), 0"""
        out = np.zeros((self.n, self.nrays(), RAY_SLOT))
        self.L.cassie_batch_get_rays.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        if self.L.cassie_batch_get_rays(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error())
        return out

    def height_scan(self):
        """[n, k] torch view (no copy) of the world z of each ray's hit, or of its end point when it hits nothing, from the last raycast()"""
        return self.torch_view('rays')[:, 1::RAY_SLOT]

    # ---- depth camera (the reference's CassieVis attach_cam / init_depth / draw_depth, example/cassietest_depth.py): one camera per batch, rendered at
    # the CURRENT state of every environment; the static geoms with each environment's own placement and terrain, and the robot's collision geoms
    def set_camera(self, name=None, body=None, pos=None, quat=None, fovy=45.0, width=64, height=64, zfar=5.0):
        """a fixed <camera> of the model by name (e.g. 'egocentric' of cassie_depth.xml), or a camera mounted on a body: pos / quat in the body frame,
        fovy the full vertical angle in degrees.  The camera looks along its -z axis with +y up.  width = 0 drops the camera.  Reallocates the rows: a
        torch_view('depth') taken before it must not be used after it."""
        if width == 0 or name is not None:
            self.L.cassie_batch_set_camera.argtypes = [C.c_void_p, C.c_char_p, C.c_int, C.c_int, C.c_double]
            rc = self.L.cassie_batch_set_camera(self.h, None if name is None else name.encode(), int(width), int(height), float(zfar))
        else:
            if body is None:
                raise ValueError('set_camera needs a camera name or a body to mount the camera on')
            p = np.ascontiguousarray(np.zeros(3) if pos is None else np.asarray(pos, dtype=np.float64).reshape(3))
            q = np.ascontiguousarray(np.array([1.0, 0, 0, 0]) if quat is None else np.asarray(quat, dtype=np.float64).reshape(4))
            self.L.cassie_batch_set_camera_mount.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_double, C.c_int, C.c_int, C.c_double]
            rc = self.L.cassie_batch_set_camera_mount(self.h, body.encode(), self._dp(p), self._dp(q), float(fovy), int(width), int(height), float(zfar))
        if rc != 0:
            raise RuntimeError(_last_error())
        self._cam_shape = (int(height), int(width)) if width else None

    def _cam_lib(self):
        L = self.L
        if not getattr(L, '_cam_bound', False):
            vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
            L.cassie_batch_set_cameras.argtypes = [vp, C.c_int, ip, dp, dp, dp, C.c_int, C.c_int, C.c_double]
            L.cassie_batch_model_camera.argtypes = [vp, C.c_char_p, ip, dp, dp, dp]
            L.cassie_batch_ncameras.argtypes = [vp]
            L.cassie_batch_set_env_cameras.argtypes = [vp, dp, dp, dp, vp]
            L.cassie_batch_get_env_cameras.argtypes = [vp, dp, dp, dp]
            L.cassie_batch_clear_env_cameras.argtypes = [vp]
            L.cassie_batch_enable_camera_geoms.argtypes = [vp, C.c_int]
            L.cassie_batch_get_camera_geoms.argtypes = [vp, ip]
            L._cam_bound = True
        return L

    def model_camera(self, name):
        """(body id, pos [3], quat [4], fovy) of a fixed <camera> of the model, e.g. 'egocentric' of cassie_depth.xml"""
        body, pos, quat, fovy = C.c_int(), np.zeros(3), np.zeros(4), C.c_double()
        if self._cam_lib().cassie_batch_model_camera(self.h, name.encode(), C.byref(body), self._dp(pos), self._dp(quat), C.byref(fovy)) != 0:
            raise RuntimeError(_last_error())
        return body.value, pos, quat, fovy.value

    def set_cameras(self, cams, width=64, height=64, zfar=5.0):
        """a set of up to CAM_MAX cameras rendered in one launch, sharing one image size and zfar.  Each entry of cams is a model camera name or
        (body, pos, quat, fovy): body a name or an id, pos / quat in the body frame, fovy the full vertical angle in degrees.  An empty list drops the
        set.  depth() and torch_view('depth') are then [n, k, height, width].  Drops the depth, geom-id and per-environment mount rows: views taken
        before it must not be used after it."""
        L = self._cam_lib()
        k = len(cams)
        body, pos, quat, fovy = np.zeros(k, dtype=np.int32), np.zeros((k, 3)), np.zeros((k, 4)), np.zeros(k)
        for i, c in enumerate(cams):
            if isinstance(c, str):
                body[i], pos[i], quat[i], fovy[i] = self.model_camera(c)
                continue
            b, p, q, f = c
            body[i] = self.name2id('body', b) if isinstance(b, str) else int(b)
            pos[i], quat[i], fovy[i] = p, q, f
        if L.cassie_batch_set_cameras(self.h, k, body.ctypes.data_as(C.POINTER(C.c_int)), self._dp(pos), self._dp(quat), self._dp(fovy),
                                      int(width), int(height), float(zfar)) != 0:
            raise RuntimeError(_last_error())
        self._cam_shape = (k, int(height), int(width)) if k else None

    def ncameras(self):
        return int(self._cam_lib().cassie_batch_ncameras(self.h))

    def set_env_cameras(self, pos=None, quat=None, fovy=None, mask=None):
        """each environment's camera mounts: pos [k, 3] or [n, k, 3] and quat [k, 4] or [n, k, 4] in each camera's body frame, fovy [k] or [n, k] in
        degrees; the body stays the set's.  A part left None is kept; mask [n]: only the selected environments change.  The first call starts every
        environment from the set's mounts.  A non-finite value, a zero quaternion or a fovy outside (0, 180) raises, and nothing changes.  Resets
        and snapshot restores leave the rows alone; a new set drops them.  torch_view('camera_env') [n, k, 8] is the device copy, read at the next
        render."""
        L, k = self._cam_lib(), self.ncameras()
        p = self._arr(pos, np.float64, (self.n, k, 3))
        q = self._arr(quat, np.float64, (self.n, k, 4))
        f = self._arr(fovy, np.float64, (self.n, k))
        m = self._arr(mask, np.uint8, (self.n,))
        ptr = lambda a: None if a is None else self._dp(a)
        if L.cassie_batch_set_env_cameras(self.h, ptr(p), ptr(q), ptr(f), None if m is None else m.ctypes.data_as(C.c_void_p)) != 0:
            raise RuntimeError(_last_error())

    def env_cameras(self):
        """(pos [n, k, 3], quat [n, k, 4], fovy [n, k]): the mount every environment's cameras see (the set's without rows)"""
        L, k = self._cam_lib(), self.ncameras()
        p, q, f = np.zeros((self.n, k, 3)), np.zeros((self.n, k, 4)), np.zeros((self.n, k))
        if L.cassie_batch_get_env_cameras(self.h, self._dp(p), self._dp(q), self._dp(f)) != 0:
            raise RuntimeError(_last_error())
        return p, q, f

    def clear_env_cameras(self):
        """back to the set's mounts in every environment"""
        if self._cam_lib().cassie_batch_clear_env_cameras(self.h) != 0:
            raise RuntimeError(_last_error())

    def enable_camera_geoms(self, on=True):
        """every render also writes the model geom id of each pixel's surface (-1: nothing within zfar); False frees the rows"""
        if self._cam_lib().cassie_batch_enable_camera_geoms(self.h, 1 if on else 0) != 0:
            raise RuntimeError(_last_error())

    def camera_geoms(self):
        """geom ids of the last render, shaped as depth(): [n, k, height, width] (set_cameras) or [n, height, width] (set_camera)"""
        shape = getattr(self, '_cam_shape', None)
        out = np.zeros((self.n,) + (shape or (0,)), dtype=np.int32)
        if shape is None or self._cam_lib().cassie_batch_get_camera_geoms(self.h, out.ctypes.data_as(C.POINTER(C.c_int))) != 0:
            raise RuntimeError(_last_error() if shape else 'no camera is set (set_camera / set_cameras)')
        return out

    def render_depth(self):
        """enqueue one depth render of every environment on the batch's stream (asynchronous), at the CURRENT state; nothing else is written"""
        self.L.cassie_batch_render_depth.argtypes = [C.c_void_p]
        if self.L.cassie_batch_render_depth(self.h) != 0:
            raise RuntimeError(_last_error())

    def depth(self):
        """[n, height, width] (set_camera) or [n, k, height, width] (set_cameras) z-depths (metres, row 0 at the top; zfar where nothing is hit) of
        the last render_depth()"""
        hw = getattr(self, '_cam_shape', None)
        out = np.zeros((self.n,) + (hw or (0, 0)))
        self.L.cassie_batch_get_depth.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        if hw is None or self.L.cassie_batch_get_depth(self.h, self._dp(out)) != 0:
            raise RuntimeError(_last_error() if hw else 'no camera is set (set_camera)')
        return out

    def query(self):
        """refresh the centre-of-mass slots of the aux rows for the CURRENT state (nothing else is written)."""
        if self.L.cassie_batch_query(self.h) != 0:
            raise RuntimeError(_last_error())

    def set_qpos(self, q):
        q = np.ascontiguousarray(q, dtype=np.float64)
        assert q.shape == (self.n, self.nq)
        self.L.cassie_batch_set_qpos(self.h, self._dp(q))

    def set_qvel(self, v):
        v = np.ascontiguousarray(v, dtype=np.float64)
        assert v.shape == (self.n, self.nv)
        self.L.cassie_batch_set_qvel(self.h, self._dp(v))

    def apply_force(self, xfrc, body_name='cassie-pelvis'):
        x = np.ascontiguousarray(np.broadcast_to(np.asarray(xfrc, dtype=np.float64), (self.n, 6)))
        return self.L.cassie_batch_apply_force(self.h, self._dp(x), body_name.encode())

    def clear_forces(self):
        self.L.cassie_batch_clear_forces(self.h)

    def set_hfield_data(self, data):
        """data: [K, nrow, ncol] (or [nrow, ncol]) normalised elevations; env e uses terrain e % K."""
        a = np.ascontiguousarray(data, dtype=np.float32)
        nrow, ncol = self.L.cassie_batch_hfield_nrow(self.h), self.L.cassie_batch_hfield_ncol(self.h)
        a = a.reshape(-1, nrow, ncol)
        if self.L.cassie_batch_set_hfielddata(self.h, a.ctypes.data_as(C.POINTER(C.c_float)), a.shape[0]) != 0:
            raise RuntimeError(_last_error())

    def get_state(self, snap=None):
        """device-resident snapshot of every row array (qpos, qvel, warm start, controller / sensor state, filters, forces, estimator, observation rows)"""
        self.L.cassie_batch_state_alloc.restype = C.c_void_p
        self.L.cassie_batch_state_alloc.argtypes = [C.c_void_p]
        self.L.cassie_batch_get_state.argtypes = [C.c_void_p, C.c_void_p]
        snap = snap or self.L.cassie_batch_state_alloc(self.h)
        if not snap or self.L.cassie_batch_get_state(self.h, C.c_void_p(snap)) != 0:
            raise RuntimeError(_last_error())
        return snap

    def set_state(self, snap, mask=None):
        m = None if mask is None else np.ascontiguousarray(mask, dtype=np.uint8)
        self.L.cassie_batch_set_state.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        if self.L.cassie_batch_set_state(self.h, C.c_void_p(snap), None if m is None else m.ctypes.data) != 0:
            raise RuntimeError(_last_error())

    def free_state(self, snap):
        self.L.cassie_batch_state_free.argtypes = [C.c_void_p, C.c_void_p]
        self.L.cassie_batch_state_free(self.h, C.c_void_p(snap))

    # ---- device-side resets: a bank of start states, restored under a device mask with no host round trip
    def _reset_lib(self):
        L = self.L
        if not getattr(L, '_reset_bound', False):
            vp = C.c_void_p
            L.cassie_batch_set_reset_bank.argtypes = [vp, vp, C.POINTER(C.c_int), C.c_int]
            L.cassie_batch_reset_bank_size.argtypes = [vp]
            L.cassie_batch_reset_where.argtypes = [vp, vp, vp]
            L.cassie_batch_forward_where.argtypes = [vp, vp]
            for n in ('set_reset_bank', 'reset_bank_size', 'reset_where', 'forward_where'):
                getattr(L, 'cassie_batch_' + n).restype = C.c_int
            L._reset_bound = True
        return L

    def set_reset_bank(self, snap, envs=None, k=None):
        """the reset bank: entry i is environment envs[i] of the snapshot `snap` (get_state of this or any batch of the same precision and model,
        of any size); envs None: the first k environments (k defaults to this batch's size).  Every call replaces the bank; snap None frees it.
        An envs index outside the snapshot or a snapshot of another precision or model raises, and the old bank is kept."""
        L = self._reset_lib()
        if snap is None:
            rc = L.cassie_batch_set_reset_bank(self.h, None, None, 0)
        elif envs is None:
            rc = L.cassie_batch_set_reset_bank(self.h, C.c_void_p(snap), None, self.n if k is None else int(k))
        else:
            e = np.ascontiguousarray(envs, dtype=np.int64).ravel()
            if e.size and (e.min() < -2 ** 31 or e.max() >= 2 ** 31):
                raise ValueError('envs must fit int32')
            e = e.astype(np.int32)
            rc = L.cassie_batch_set_reset_bank(self.h, C.c_void_p(snap), e.ctypes.data_as(C.POINTER(C.c_int)), int(e.size))
        if rc != 0:
            raise RuntimeError(_last_error())

    def reset_bank_size(self):
        return int(self._reset_lib().cassie_batch_reset_bank_size(self.h))

    def _device_rows(self, t, what, dtypes):
        import torch
        if not isinstance(t, torch.Tensor):
            raise TypeError('%s must be a CUDA torch tensor, not %s' % (what, type(t).__name__))
        if not t.is_cuda or t.device.index != self.device:
            raise ValueError('%s must be on cuda:%d (the batch\'s device), not %s' % (what, self.device, t.device))
        if t.dtype not in dtypes or t.numel() != self.n or not t.is_contiguous():
            raise ValueError('%s must be a contiguous tensor of %d elements of %s, not %s %s' % (what, self.n, ' / '.join(str(d) for d in dtypes), t.dtype, tuple(t.shape)))
        return t

    def _mask_ptr(self, mask, what):
        import torch
        m = self._device_rows(mask, what, (torch.bool, torch.uint8))
        return (m.view(torch.uint8) if m.dtype == torch.bool else m).data_ptr()   # bool is one byte per element: reinterpreted, not copied

    def reset_where(self, done, entry=None):
        """environments with done[e] set take bank entry entry[e] mod K (entry None: e mod K), as set_state would restore that entry; the others are
        untouched.  done: CUDA bool / uint8 tensor [n]; entry: CUDA int32 / int64 tensor [n] (int64 is converted, and the int32 copy kept until the
        next call so that it outlives the launch).  One launch on the batch's stream: no host synchronisation, capturable in a CUDA graph.

        Stream rule (as torch_view's): done and entry are written on torch's stream and must be ordered before the batch's stream, so either run the
        batch on torch's stream (set_stream(torch.cuda.current_stream().cuda_stream)) or synchronise before the call."""
        import torch
        L = self._reset_lib()
        mp = self._mask_ptr(done, 'done')
        ep = None
        if entry is not None:
            e = self._device_rows(entry, 'entry', (torch.int32, torch.int64))
            if e.dtype == torch.int64:
                e = e.to(torch.int32)
            self._entry_tmp = e
            ep = e.data_ptr()
        if L.cassie_batch_reset_where(self.h, C.c_void_p(mp), None if ep is None else C.c_void_p(ep)) != 0:
            raise RuntimeError(_last_error())

    def forward_where(self, mask):
        """mj_forward for the environments with mask[e] set (CUDA bool / uint8 tensor [n]), each on its own model rows; the others are untouched.
        Asynchronous and capturable like reset_where, with its stream rule: e.g. reset_where, noise written into torch_view('qpos') / ('qvel') of the
        reset environments, forward_where."""
        L = self._reset_lib()
        if L.cassie_batch_forward_where(self.h, C.c_void_p(self._mask_ptr(mask, 'mask'))) != 0:
            raise RuntimeError(_last_error())

    # ---- loop closure: qpos and qvel projected onto the legs' connect equalities (rules in include/cassie_b200.h, DESIGN.md section 3)
    LOOP_TOL = {FP64: 1e-12, FP32: 1e-6}   # metres: fp32 kinematics reaches ~5e-7 at best, so 1e-6 converges in 2-4 steps from 0.05 rad of noise

    def close_loops(self, mask=None, max_iter=20, tol=None):
        """close the loops of the environments with mask[e] set (CUDA bool / uint8 tensor [n]; None: every environment): the rod, tarsus, crank and
        plantar-rod coordinates are moved until max |p1 - p2| <= tol (None: LOOP_TOL of the precision) or max_iter damped Gauss-Newton steps, and their
        velocities projected so that J qvel ~ 0; everything else is held bitwise.  An environment that does not converge keeps qpos and qvel.  One
        launch on the batch's stream, capturable in a CUDA graph after the first call (which allocates the status rows), with reset_where's stream
        rule.  It writes qpos, qvel and loop_status() only: follow it with forward_where(mask) to refresh the observation, sensors and frames"""
        L = self.L
        L.cassie_batch_close_loops.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double]
        mp = None if mask is None else C.c_void_p(self._mask_ptr(mask, 'mask'))
        if L.cassie_batch_close_loops(self.h, mp, int(max_iter), float(self.LOOP_TOL[self.precision] if tol is None else tol)) != 0:
            raise RuntimeError(_last_error())

    def loop_status(self):
        """the status rows of the last close_loops, as numpy arrays [n]: residual (max |p1 - p2| in metres after the launch; for a failure, that of the
        unchanged pose), iterations (0: already closed, -1: not converged) and vel_residual (max |J qvel| after the launch); environments outside the
        last mask keep the values of their last selection (zero before it)"""
        out = dict(residual=np.zeros(self.n), iterations=np.zeros(self.n, dtype=np.int32), vel_residual=np.zeros(self.n))
        self.L.cassie_batch_get_loop_status.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int), C.POINTER(C.c_double)]
        if self.L.cassie_batch_get_loop_status(self.h, self._dp(out['residual']), out['iterations'].ctypes.data_as(C.POINTER(C.c_int)), self._dp(out['vel_residual'])) != 0:
            raise RuntimeError(_last_error())
        return out

    # ---- inverse kinematics: free coordinates posed to per-environment frame targets (rules in include/cassie_b200.h, DESIGN.md section 3)
    IK_TOL = {FP64: 1e-10, FP32: 1e-5}    # metres and radians: fp32 kinematics reaches ~1e-6 at best; fp64 reaches 1e-10 in 4-6 steps from a standing pose

    def set_ik(self, names, kinds, frames=None, weights=None):
        """the target list (at most IK_MAX): body or site names with kinds FRAME_BODY / FRAME_SITE, frames IK_WORLD / IK_ROOT (None: all world), weights
        [k][6] for the position rows x, y, z and the orientation rows about the target's x, y, z (None: all 1; 0 drops a row).  [] drops the list.  It
        allocates the target rows torch_view('ik_targets') [n, IK_MAX, 16] (position 3, quaternion 4, linear velocity 3, angular velocity 3, pad) and the
        status rows torch_view('ik') [n, 8], zero"""
        names = list(names)
        k = len(names)
        kinds = [int(x) for x in kinds]
        frames = [IK_WORLD] * k if frames is None else [int(x) for x in frames]
        w = np.ones((k, 6)) if weights is None else np.array(weights, dtype=np.float64).reshape(k, 6)
        if len(kinds) != k or len(frames) != k:
            raise ValueError('one kind and one frame per target name')
        arr = (C.c_char_p * max(1, k))(*[n.encode() for n in names])
        ks, fs = (C.c_int * max(1, k))(*kinds), (C.c_int * max(1, k))(*frames)
        w = np.ascontiguousarray(w)
        self.L.cassie_batch_set_ik.argtypes = [C.c_void_p, C.POINTER(C.c_char_p), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_double), C.c_int]
        if self.L.cassie_batch_set_ik(self.h, arr, ks, fs, self._dp(w), k) != 0:
            raise RuntimeError(_last_error())

    def solve_ik(self, mask=None, max_iter=100, tol=None, velocities=False):
        """pose the environments with mask[e] set (CUDA bool / uint8 tensor [n]; None: every environment) to their rows of torch_view('ik_targets'):
        Levenberg-Marquardt steps on the free coordinates (motors and the loops' passive joints) from the current qpos, loops closed and joint ranges
        held, until every weighted row is within tol (None: IK_TOL of the precision) or the steps stall or max_iter runs out; velocities=True also fits
        the free qvel to the rows' velocities.  One launch on the batch's stream, capturable in a CUDA graph; it writes qpos, qvel and ik_status() only:
        follow it with forward_where(mask)"""
        L = self.L
        L.cassie_batch_solve_ik.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_int]
        mp = None if mask is None else C.c_void_p(self._mask_ptr(mask, 'mask'))
        if L.cassie_batch_solve_ik(self.h, mp, int(max_iter), float(self.IK_TOL[self.precision] if tol is None else tol), 1 if velocities else 0) != 0:
            raise RuntimeError(_last_error())

    def ik_status(self):
        """the status rows of the last solve_ik as numpy arrays [n], named as IK_STATUS: pos_residual (m), ori_residual (rad), loop_residual (m),
        iterations, outcome (1 reached, 2 best effort, -1 kept), jeq_qvel (max |J_eq qvel|), vel_residual, at_bound (free joints at a range bound);
        environments outside the last mask keep their values (zero before their first selection)"""
        st = np.zeros((self.n, IK_SLOT))
        self.L.cassie_batch_get_ik_status.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        if self.L.cassie_batch_get_ik_status(self.h, self._dp(st)) != 0:
            raise RuntimeError(_last_error())
        out = {k: st[:, i].copy() for i, k in enumerate(IK_STATUS)}
        for k in ('iterations', 'outcome', 'at_bound'):
            out[k] = out[k].astype(np.int32)
        return out

    def set_timestep(self, dt):
        self.L.cassie_batch_set_timestep.argtypes = [C.c_void_p, C.c_double]
        if self.L.cassie_batch_set_timestep(self.h, float(dt)) != 0:
            raise RuntimeError(_last_error())

    def row_width(self, field):
        """row width (elements) of a device array: qpos 36 (44 with the extra free body), qvel 32 (40), pd 52, obs 112, xfrc 8, aux 64"""
        self.L.cassie_batch_row_width.argtypes = [C.c_void_p, C.c_char_p]
        return int(self.L.cassie_batch_row_width(self.h, field.encode()))

    def counters(self):
        out = np.zeros((self.n, 8), dtype=np.int32)
        self.L.cassie_batch_get_counters(self.h, out.ctypes.data_as(C.POINTER(C.c_int)))
        return out

    def debug_dump(self, env=0):
        out = np.zeros(3600)
        k = self.L.cassie_batch_debug_dump(self.h, env, self._dp(out), out.size)
        return out if k > 0 else None

    def launch_count(self):
        return int(self.L.cassie_batch_launch_count(self.h))

    def device_ptr(self, field):
        return self.L.cassie_batch_device_ptr(self.h, field.encode())

    def set_stream(self, cuda_stream_ptr):
        self.L.cassie_batch_set_stream(self.h, C.c_void_p(cuda_stream_ptr))

    def torch_view(self, field):
        """zero-copy torch tensor over a device state array (qpos [n,36], qvel [n,32], pd [n,52], obs [n,112], aux [n,64], frames [n, nframes * 20],
        frame_jac [n, 240], dyn [n, DYN_WIDTH] laid out as DYN, rays [n, k * RAY_SLOT], acc [n, acc_width(nframes)] laid out as ACC, depth [n, height, width] (set_camera) or [n, k, height, width] (set_cameras),
        terrain [n] int32: each environment's bank entry, read mod K at the next launch; set_env_hfield first; actuators [n, 40]: lo[10], hi[10], wmax[10]
        in rad/s, delay[10], read at the next launch; set_env_actuators first; mechanics [n, 192]: body_inertia[32][3], armature[32], stiffness[32],
        qpos_spring[32] per main-tree dof (the springs of hinge dofs only are read), read at the next launch; set_env_mechanics first; contact [n, 256]:
        32 slots of 8 -- solref[2], solimp[5], solmix -- one per device collision geom (moving 0..15, static 16..31; unused slots zero), read at the next
        launch; set_env_contact first; applied [n, 232]: xfrc_applied[32][6] in model body order, then qfrc_applied[40] by dof column (main tree 0..31,
        the extra free body 32..37), read at the next launch; set_applied_forces or enable_applied_forces first; trace [n, T, k]: the per-tick trace of
        the last step launch, slot s of every environment, written by step launches only; set_trace first; inv_qacc [n, qvel width]: the qacc of
        compute_inverse(None), column = dof; inv [n, INV_WIDTH] laid out as INV; both allocated by the first request; contacts [n, CON_WIDTH]: the contact
        lists of the last step / forward launch, a header and CON_MAX slots laid out as CON; enable_contacts first; camera_env [n, k, CAMENV_SLOT]: the
        per-environment camera mounts pos[3], quat[4], fovy in degrees, read at the next render; set_env_cameras first; camera_geom [n, k, height, width]
        int32 (shaped as depth for set_camera): the geom ids of the last render; enable_camera_geoms and render_depth first; sensors [n, 52] laid out as
        SN, read at the next launch; sensor_rng [n, 4] int32: key lo, hi, counter lo, hi; set_env_sensors first for both; loops [n, 4]: the status
        rows of close_loops -- residual, iterations, max |J qvel|, pad; close_loops first; ik_targets [n, IK_MAX, 16]: the targets of solve_ik, written by
        the caller; ik [n, 8]: its status rows laid out as IK_STATUS; set_ik first for both).  set_frames /
        set_rays / set_camera reallocate the frame, acceleration, ray and depth rows: a view taken before them must not be used after them.  The dynamics rows stay put once compute_dynamics() has allocated them.

        The arrays are written on the batch's stream.  Unless that stream is torch's current stream (set_stream(torch.cuda.current_stream().cuda_stream)),
        call sync() before reading the view: torch ops on another stream are not ordered after an in-flight step."""
        import torch
        self.L.cassie_batch_row_width.argtypes = [C.c_void_p, C.c_char_p]
        width = self.L.cassie_batch_row_width(self.h, field.encode())
        ptr = self.device_ptr(field)
        if width <= 0 or not ptr:
            raise RuntimeError('no device rows for %r (frames: set_frames first; frame_jac: frame_jacobian first; dyn: compute_dynamics first; rays: raycast first; acc: enable_accelerations first; depth: render_depth first; terrain: set_env_hfield first; actuators: set_env_actuators first; mechanics: set_env_mechanics first; contact: set_env_contact first; applied: enable_applied_forces first; trace: set_trace first; contacts: enable_contacts first; camera_env: set_env_cameras first; camera_geom: enable_camera_geoms and render_depth first; sensors, sensor_rng: set_env_sensors first; loops: close_loops first; ik_targets, ik: set_ik first)' % field)
        dt, isz, ts = (np.float32, 4, '<f4') if self.precision == FP32 else (np.float64, 8, '<f8')
        if field in ('terrain', 'camera_geom', 'sensor_rng'):
            ts = '<i4'

        class _Arr:
            pass
        a = _Arr()
        a.__cuda_array_interface__ = dict(shape=(self.n, width), typestr=ts, data=(ptr, False), version=2)
        t = torch.as_tensor(a, device='cuda')
        if field == 'terrain':
            return t.view(self.n)
        if field == 'trace':
            return t.view(self.n, *self._trace_shape)
        if field == 'camera_env':
            return t.view(self.n, -1, CAMENV_SLOT)
        if field == 'ik_targets':
            return t.view(self.n, IK_MAX, IK_TARGET_WIDTH)
        return t.view(self.n, *self._cam_shape) if field in ('depth', 'camera_geom') else t


class joint_filter_t(C.Structure):
    """the joint encoders' IIR filter state, as the C struct"""
    _fields_ = [('x', C.c_double * 4), ('y', C.c_double * 3)]


class drive_filter_t(C.Structure):
    """the drive encoders' FIR taps: int x[9] as in the C struct (the reference's ctypes file declares doubles here)"""
    _fields_ = [('x', C.c_int * 9)]


class cassie_user_in_t(C.Structure):
    _fields_ = [('torque', C.c_double * 10), ('telemetry', C.c_short * 9)]


class elmo_out_t(C.Structure):
    _fields_ = [('statusWord', C.c_ushort), ('position', C.c_double), ('velocity', C.c_double), ('torque', C.c_double), ('driveTemperature', C.c_double),
                ('dcLinkVoltage', C.c_double), ('torqueLimit', C.c_double), ('gearRatio', C.c_double)]


class cassie_joint_out_t(C.Structure):
    _fields_ = [('position', C.c_double), ('velocity', C.c_double)]


class cassie_leg_out_t(C.Structure):
    _fields_ = [(n, elmo_out_t) for n in ('hipRollDrive', 'hipYawDrive', 'hipPitchDrive', 'kneeDrive', 'footDrive')] + \
               [(n, cassie_joint_out_t) for n in ('shinJoint', 'tarsusJoint', 'footJoint')] + \
               [('medullaCounter', C.c_ubyte), ('medullaCpuLoad', C.c_ushort), ('reedSwitchState', C.c_bool)]


class battery_out_t(C.Structure):
    _fields_ = [('dataGood', C.c_bool), ('stateOfCharge', C.c_double), ('voltage', C.c_double * 12), ('current', C.c_double), ('temperature', C.c_double * 4)]


class radio_out_t(C.Structure):
    _fields_ = [('radioReceiverSignalGood', C.c_bool), ('receiverMedullaSignalGood', C.c_bool), ('channel', C.c_double * 16)]


class target_pc_out_t(C.Structure):
    _fields_ = [('etherCatStatus', C.c_int * 6), ('etherCatNotifications', C.c_int * 21), ('taskExecutionTime', C.c_double), ('overloadCounter', C.c_uint), ('cpuTemperature', C.c_double)]


class vectornav_out_t(C.Structure):
    _fields_ = [('dataGood', C.c_bool), ('vpeStatus', C.c_ushort), ('pressure', C.c_double), ('temperature', C.c_double), ('magneticField', C.c_double * 3),
                ('angularVelocity', C.c_double * 3), ('linearAcceleration', C.c_double * 3), ('orientation', C.c_double * 4)]


class cassie_pelvis_out_t(C.Structure):
    _fields_ = [('targetPc', target_pc_out_t), ('battery', battery_out_t), ('radio', radio_out_t), ('vectorNav', vectornav_out_t), ('medullaCounter', C.c_ubyte),
                ('medullaCpuLoad', C.c_ushort), ('bleederState', C.c_bool), ('leftReedSwitchState', C.c_bool), ('rightReedSwitchState', C.c_bool), ('vtmTemperature', C.c_double)]


class cassie_out_t(C.Structure):
    _fields_ = [('pelvis', cassie_pelvis_out_t), ('leftLeg', cassie_leg_out_t), ('rightLeg', cassie_leg_out_t), ('isCalibrated', C.c_bool), ('messages', C.c_short * 4)]


assert C.sizeof(cassie_out_t) == 1336 and C.sizeof(cassie_user_in_t) == 104


class CassieState:
    """cassie_state_t (reference: example/cassiemujoco.py CassieState): a full dynamic-state snapshot of a CassieSim"""

    def __init__(self):
        self.L = lib()
        self.s = self.L.cassie_state_alloc()

    def time(self):
        return self.L.cassie_state_time(self.s)[0]

    def qpos(self):
        return np.array(self.L.cassie_state_qpos(self.s)[:35])

    def qvel(self):
        return np.array(self.L.cassie_state_qvel(self.s)[:32])

    def set_time(self, t):
        self.L.cassie_state_time(self.s)[0] = t

    def set_qpos(self, q):
        p = self.L.cassie_state_qpos(self.s)
        for i in range(len(q)):
            p[i] = q[i]

    def set_qvel(self, v):
        p = self.L.cassie_state_qvel(self.s)
        for i in range(len(v)):
            p[i] = v[i]

    def close(self):
        if getattr(self, 's', None):
            self.L.cassie_state_free(self.s)
            self.s = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class CassieSim:
    """Legacy single-environment object (reference: example/cassiemujoco.py:31-173), stepped by the same CUDA kernels."""

    def __init__(self, modelfile=None, reinit=True):   # the reference wrapper always passes reinit=True (example/cassiemujoco.py:44)
        self.L = lib()
        path = modelfile or model_path()
        self.c = self.L.cassie_sim_init(path.encode(), bool(reinit))
        if not self.c:
            raise RuntimeError('cassie_sim_init failed: ' + _last_error())
        self.nq, self.nv = self.L.cassie_sim_nq(self.c), self.L.cassie_sim_nv(self.c)

    def step_pd(self, u):
        y = state_out_t()
        self.L.cassie_sim_step_pd(self.c, C.byref(y), C.byref(u))
        return y

    def time(self):
        return self.L.cassie_sim_time(self.c)[0]

    def mj_name2id(self, obj_type, name):
        """id of a named body, joint, geom, site or camera, or -1 (reference: example/cassiemujoco.py:821-822)"""
        self.L.cassie_sim_mj_name2id.argtypes = [C.c_void_p, C.c_char_p, C.c_char_p]
        self.L.cassie_sim_mj_name2id.restype = C.c_int
        return int(self.L.cassie_sim_mj_name2id(self.c, obj_type.encode(), name.encode()))

    def qpos(self):
        return np.array(self.L.cassie_sim_qpos(self.c)[:self.nq])

    def qvel(self):
        return np.array(self.L.cassie_sim_qvel(self.c)[:self.nv])

    def set_time(self, t):
        self.L.cassie_sim_time(self.c)[0] = t

    def set_qpos(self, qpos):
        p = self.L.cassie_sim_qpos(self.c)
        for i in range(min(len(qpos), self.nq)):
            p[i] = qpos[i]

    def set_qvel(self, qvel):
        p = self.L.cassie_sim_qvel(self.c)
        for i in range(min(len(qvel), self.nv)):
            p[i] = qvel[i]

    def apply_force(self, xfrc, body_name='cassie-pelvis'):
        a = (C.c_double * 6)(*[float(x) for x in xfrc])
        self.L.cassie_sim_apply_force(self.c, a, body_name.encode())

    def clear_forces(self):
        self.L.cassie_sim_clear_forces(self.c)

    def full_reset(self):
        self.L.cassie_sim_full_reset(self.c)

    # ---- the verbs around the hot path (reference: example/cassiemujoco.py:64-173)
    def step(self, u):
        """torque-level step: u = cassie_user_in_t; returns the cassie_out_t of this tick"""
        y = cassie_out_t()
        self.L.cassie_sim_step(self.c, C.addressof(y), C.addressof(u))
        return y

    def step_pd_no2khz(self, u):
        y = state_out_t()
        self.L.cassie_sim_step_pd_no2khz(self.c, C.byref(y), C.byref(u))
        return y

    def get_cassie_out(self):
        self.L.cassie_sim_get_cassie_out.restype = cassie_out_t
        self.L.cassie_sim_get_cassie_out.argtypes = [C.c_void_p]
        return self.L.cassie_sim_get_cassie_out(self.c)

    def timestep(self):
        return self.L.cassie_sim_timestep(self.c)[0]

    def set_timestep(self, dt):
        self.L.cassie_sim_set_timestep(self.c, float(dt))

    def forward(self):
        return self.L.cassie_sim_forward(self.c)

    def hold(self):
        self.L.cassie_sim_hold(self.c)

    def release(self):
        self.L.cassie_sim_release(self.c)

    def get_state(self, s=None):
        s = s or CassieState()
        self.L.cassie_get_state(self.c, s.s)
        return s

    def set_state(self, s):
        self.L.cassie_set_state(self.c, s.s)

    def duplicate(self):
        d = CassieSim.__new__(CassieSim)
        d.L = self.L
        d.c = self.L.cassie_sim_duplicate(self.c)
        if not d.c:
            raise RuntimeError('cassie_sim_duplicate failed: ' + _last_error())
        d.nq, d.nv = self.nq, self.nv
        return d

    def copy(self, src):
        self.L.cassie_sim_copy(self.c, src.c)

    # ---- model constants, named as in the reference wrapper (example/cassiemujoco.py:380-610)
    def params(self):
        p = (C.c_int * 6)()
        self.L.cassie_sim_params(self.c, p)
        return list(p)

    def _marr(self, fn, n):
        return np.array(fn(self.c)[:n])

    def get_dof_damping(self, name=None):
        if name:
            return np.array(self.L.cassie_sim_get_dof_name_damping(self.c, name.encode())[:self.L.cassie_sim_get_joint_num_dof(self.c, name.encode())])
        return self._marr(self.L.cassie_sim_dof_damping, self.nv)

    def get_body_mass(self, name=None):
        if name:
            return self.L.cassie_sim_get_body_name_mass(self.c, name.encode())
        return self._marr(self.L.cassie_sim_body_mass, self.params()[4])

    def get_body_ipos(self, name=None):
        if name:
            return np.array(self.L.cassie_sim_get_body_name_ipos(self.c, name.encode())[:3])
        return self._marr(self.L.cassie_sim_body_ipos, 3 * self.params()[4])

    def get_body_pos(self, name):
        """the body's position in its parent frame (reference: example/cassiemujoco.py:437-442)"""
        ptr = self.L.cassie_sim_get_body_name_pos(self.c, name.encode())
        if not ptr:
            raise RuntimeError(_last_error())
        return np.array(ptr[:3])

    def get_geom_friction(self, name=None):
        if name:
            return np.array(self.L.cassie_sim_get_geom_name_friction(self.c, name.encode())[:3])
        ng = self.params()[5]
        return self._marr(self.L.cassie_sim_geom_friction, 3 * ng).reshape(ng, 3)

    @staticmethod
    def _carr(data):
        a = np.ascontiguousarray(data, dtype=np.float64).ravel()
        return (C.c_double * a.size)(*a)

    def set_dof_damping(self, data, name=None):
        if name:
            self.L.cassie_sim_set_dof_name_damping(self.c, name.encode(), self._carr(np.atleast_1d(data)))
        else:
            assert len(data) == self.nv
            self.L.cassie_sim_set_dof_damping(self.c, self._carr(data))

    def set_body_mass(self, data, name=None):
        if name is None:
            assert len(data) == self.params()[4]
            self.L.cassie_sim_set_body_mass(self.c, self._carr(data))
        else:
            self.L.cassie_sim_set_body_name_mass(self.c, name.encode(), float(data))

    # ---- the controller-stage state (reference: example/cassiemujoco.py:132-161, 780-813)
    def _act_lib(self):
        L = self.L
        if not getattr(L, '_sim_act_bound', False):
            vp, dp, ip = C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_int)
            for n, a in (('cassie_sim_torque_delay', [vp, dp]), ('cassie_sim_set_torque_delay', [vp, dp]), ('cassie_sim_get_joint_filter', [vp, dp, dp]),
                         ('cassie_sim_set_joint_filter', [vp, dp, dp]), ('cassie_sim_get_drive_filter', [vp, ip]), ('cassie_sim_set_drive_filter', [vp, ip])):
                getattr(L, n).argtypes = a
                getattr(L, n).restype = None
            L.cassie_sim_joint_filter.argtypes = L.cassie_sim_drive_filter.argtypes = L.cassie_sim_ctrl.argtypes = [vp]
            L.cassie_sim_joint_filter.restype = C.POINTER(joint_filter_t)
            L.cassie_sim_drive_filter.restype = C.POINTER(drive_filter_t)
            L.cassie_sim_ctrl.restype = dp
            L._sim_act_bound = True
        return L

    def ctrl(self):
        """the ctrl [nu] the last physics step applied"""
        return self._act_lib().cassie_sim_ctrl(self.c)[:NU]

    def set_ctrl(self, ctrl):
        """writes through cassie_sim_ctrl, as the reference does; the next step overwrites it (the delay line's output is what is applied)"""
        p = self._act_lib().cassie_sim_ctrl(self.c)
        for i in range(NU):
            p[i] = ctrl[i]

    def get_joint_filter(self):
        """a pointer to the joint_filter_t[6] mirror, indexable as an array of filters (writes are uploaded before the next step)"""
        return self._act_lib().cassie_sim_joint_filter(self.c)

    def set_joint_filter(self, x, y):
        """x [6 * 4], y [6 * 3]"""
        x_arr, y_arr = (C.c_double * 24)(*x), (C.c_double * 18)(*y)
        self._act_lib().cassie_sim_set_joint_filter(self.c, C.cast(x_arr, C.POINTER(C.c_double)), C.cast(y_arr, C.POINTER(C.c_double)))

    def get_drive_filter(self):
        """a pointer to the drive_filter_t[10] mirror (int x[9] each), indexable as an array of filters"""
        return self._act_lib().cassie_sim_drive_filter(self.c)

    def set_drive_filter(self, x):
        """x [10 * 9] integers"""
        x_arr = (C.c_int * 90)(*[int(v) for v in x])
        self._act_lib().cassie_sim_set_drive_filter(self.c, C.cast(x_arr, C.POINTER(C.c_int)))

    def get_torque_delay(self):
        """the torque delay line [10, 6] (motor by delay slot, slot 0 newest)"""
        t = (C.c_double * 60)()
        self._act_lib().cassie_sim_torque_delay(self.c, t)
        return np.array(t[:]).reshape((10, 6))

    def set_torque_delay(self, data):
        t = (C.c_double * 60)(*np.asarray(data, dtype=np.float64).flatten())
        self._act_lib().cassie_sim_set_torque_delay(self.c, C.cast(t, C.POINTER(C.c_double)))

    def set_body_pos(self, name, data):
        """moves the body in its parent frame from the next step on (reference: example/cassiemujoco.py:563-570); call set_const for the
        mj_setConst constants, as with the reference"""
        assert len(data) == 3
        self.L.cassie_sim_set_body_name_pos(self.c, name.encode(), self._carr(data))

    def set_body_ipos(self, data, name=None):
        if name:
            assert len(data) == 3
            self.L.cassie_sim_set_body_name_ipos(self.c, name.encode(), self._carr(data))
        else:
            assert len(data) == 3 * self.params()[4]
            self.L.cassie_sim_set_body_ipos(self.c, self._carr(data))

    def set_geom_friction(self, data, name=None):
        if name is None:
            assert np.size(data) == 3 * self.params()[5]
            self.L.cassie_sim_set_geom_friction(self.c, self._carr(data))
        else:
            assert len(data) == 3
            self.L.cassie_sim_set_geom_name_friction(self.c, name.encode(), self._carr(data))

    def set_const(self):
        self.L.cassie_sim_set_const(self.c)

    def get_hfield_size(self):
        """the height field's size [x half-extent, y half-extent, elevation scale, base thickness] (reference: example/cassiemujoco.py:741-746)"""
        ptr = self.L.cassie_sim_get_hfield_size(self.c)
        if not ptr:
            raise RuntimeError(_last_error())
        return np.array(ptr[:4])

    def set_hfield_size(self, data):
        """applied at the next step (reference: example/cassiemujoco.py:768-776)"""
        assert len(data) == 4
        self.L.cassie_sim_set_hfield_size(self.c, (C.c_double * 4)(*[float(x) for x in data]))

    def just_set_const(self):
        self.L.cassie_sim_just_set_const(self.c)

    # ---- read-only queries, named as in the reference wrapper (example/cassiemujoco.py:214-306, 815-819)
    def _vec(self, fn, n):
        a = (C.c_double * n)()
        fn(self.c, a)
        return np.array(a[:])

    def foot_forces_raw(self):
        return self._vec(self.L.cassie_sim_foot_forces, 12)

    def get_foot_forces(self):
        f = self.foot_forces_raw()
        return float(np.sqrt((f[0:3] ** 2).sum())), float(np.sqrt((f[6:9] ** 2).sum()))

    def get_heeltoe_forces(self):
        t, h = (C.c_double * 6)(), (C.c_double * 6)()
        self.L.cassie_sim_heeltoe_forces(self.c, t, h)
        return np.array(t[:]), np.array(h[:])

    def check_collision(self, geom_group):
        return bool(self.L.cassie_sim_geom_collision(self.c, int(geom_group)))

    def foot_pos(self):
        return list(self._vec(self.L.cassie_sim_foot_positions, 6))

    def foot_vel(self, vel):
        vel[:12] = self._vec(self.L.cassie_sim_foot_velocities, 12)

    def center_of_mass_position(self):
        return list(self._vec(self.L.cassie_sim_cm_position, 3))

    def center_of_mass_velocity(self):
        return list(self._vec(self.L.cassie_sim_cm_velocity, 3))

    def angular_momentum(self):
        return list(self._vec(self.L.cassie_sim_angular_momentum, 3))

    # ---- frames (example/cassiemujoco.py:124-130, 184-214, 254-270, 694-721): what the last step / forward left behind; the Jacobians are taken at
    # the current state.  An unknown name raises (the reference indexes its arrays with -1)
    def _ptr(self, fn, name, n):
        fn.restype = C.POINTER(C.c_double)
        fn.argtypes = [C.c_void_p, C.c_char_p]
        p = fn(self.c, name.encode())
        if not p:
            raise KeyError(name)
        return np.array(p[:n])

    def _named(self, fn, name, n):
        a = (C.c_double * n)()
        fn.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.c_char_p]
        fn(self.c, a, name.encode())
        return np.array(a[:])

    def xpos(self, body_name):
        return self._ptr(self.L.cassie_sim_xpos, body_name, 3)

    def xquat(self, body_name):
        return self._ptr(self.L.cassie_sim_xquat, body_name, 4)

    def get_site_xpos(self, name):
        return self._ptr(self.L.cassie_sim_site_xpos, name, 3)

    def sense_ground(self):
        """the six rangefinders (example/cassiemujoco.py:175-181): distance along each rangefinder site's z axis to the static terrain, capped at the
        sensor's cutoff, -1 for no hit"""
        percept = (C.c_double * 6)()
        self.L.cassie_sim_read_rangefinder.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        self.L.cassie_sim_read_rangefinder.restype = None
        self.L.cassie_sim_read_rangefinder(self.c, percept)
        return np.array(percept[:6])

    def get_site_quat(self, name):
        a = (C.c_double * 4)()
        self.L.cassie_sim_site_xquat.argtypes = [C.c_void_p, C.c_char_p, C.POINTER(C.c_double)]
        self.L.cassie_sim_site_xquat(self.c, name.encode(), a)
        return a[:4]

    def qacc(self):
        """qacc of the last step / forward (nv entries)"""
        self.L.cassie_sim_qacc.restype = C.POINTER(C.c_double)
        self.L.cassie_sim_qacc.argtypes = [C.c_void_p]
        return np.array(self.L.cassie_sim_qacc(self.c)[:self.nv])

    def get_body_acceleration(self, accel, body_name):
        """cacc of the body ([angular; linear], com-based) after the last step / forward into accel[6]"""
        accel[:6] = self._named(self.L.cassie_sim_body_acceleration, body_name, 6)

    def foot_quat(self, quat):
        """the right-foot-middle site's quaternion into quat[4] (cassie_sim_foot_orient)"""
        a = (C.c_double * 4)()
        self.L.cassie_sim_foot_orient.argtypes = [C.c_void_p, C.POINTER(C.c_double)]
        self.L.cassie_sim_foot_orient.restype = None
        self.L.cassie_sim_foot_orient(self.c, a)
        quat[:4] = a[:4]

    def body_vel(self, vel, body_name):
        """cvel of the body ([angular; linear], com-based) into vel[6]; cassie_sim_body_velocities (the reference wrapper names a function its
        library does not export)"""
        vel[:6] = self._named(self.L.cassie_sim_body_velocities, body_name, 6)

    def get_body_contact_force(self, force, body_name):
        force[:6] = self._named(self.L.cassie_sim_body_contact_force, body_name, 6)

    def get_jacobian(self, name):
        return self._named(self.L.cassie_sim_get_jacobian, name, 3 * self.nv)

    def _jac_full(self, fn, name):
        p, r = (C.c_double * (3 * self.nv))(), (C.c_double * (3 * self.nv))()
        fn.argtypes = [C.c_void_p, C.POINTER(C.c_double), C.POINTER(C.c_double), C.c_char_p]
        fn(self.c, p, r, name.encode())
        return np.array(p[:]), np.array(r[:])

    def get_jacobian_full(self, name):
        return self._jac_full(self.L.cassie_sim_get_jacobian_full, name)

    def get_jacobian_full_site(self, name):
        return self._jac_full(self.L.cassie_sim_get_jacobian_full_site, name)

    def get_object_relative_pose(self, pose1, pose2, relative_pose):
        """pose 2 ([pos3, quat4]) in the frame of pose 1, into relative_pose[7]"""
        d = C.POINTER(C.c_double)
        a = [(C.c_double * k)(*v) for k, v in ((3, pose1[:3]), (4, pose1[3:7]), (3, pose2[:3]), (4, pose2[3:7]))]
        pos, quat = (C.c_double * 3)(), (C.c_double * 4)()
        self.L.cassie_sim_relative_pose.argtypes = [d] * 6
        self.L.cassie_sim_relative_pose(*a, pos, quat)
        relative_pose[:3] = pos[:]
        relative_pose[3:7] = quat[:]

    # ---- dynamics at the current state (example/cassiemujoco.py:292-375): one dynamics launch each
    def _dyn(self, fn, *sizes):
        bufs = [(C.c_double * k)() for k in sizes]
        fn.argtypes = [C.c_void_p] + [C.POINTER(C.c_double)] * len(sizes)
        fn.restype = None
        fn(self.c, *bufs)
        return [np.array(b[:]) for b in bufs]

    def centroid_inertia(self):
        """3 x 3 rotational inertia about the centre of mass in the pelvis frame, flattened (9 values), with the reference's formula"""
        return list(self._dyn(self.L.cassie_sim_centroid_inertia, 9)[0])

    def full_mass_matrix(self):
        """the 32 x 32 mass matrix of the robot's dofs"""
        return self._dyn(self.L.cassie_sim_full_mass_matrix, 32 * 32)[0].reshape(32, 32)

    def constraint_jacobian(self):
        """[6, 32]: the rows of the left and right achilles-rod connects"""
        return self._dyn(self.L.cassie_sim_loop_constraint_info, 6 * 32, 6)[0].reshape(6, 32)

    def constraint_error(self):
        """[6, 1]: their position errors"""
        return self._dyn(self.L.cassie_sim_loop_constraint_info, 6 * 32, 6)[1].reshape(6, 1)

    def minimal_mass_matrix(self):
        """16 x 16 mass matrix of the floating base and the 10 motors: the full matrix projected onto these independent coordinates through the
        achilles constraints, as the reference's wrapper does it.  The dependent coordinates (knee, shin, tarsus, heel-spring side of each leg's
        four-bar) follow from the independent ones by the least-squares solution G of J_dep G = -J_ind; with P = [I; G], M_min = P' M P.  The
        constraint Jacobian's floating-base columns are zeroed and so is every entry below 1e-5 (negative ones too), like the reference."""
        ind = [0, 1, 2, 3, 4, 5, 6, 7, 8, 12, 18, 19, 20, 21, 25, 31]
        dep = [9, 10, 11, 14, 22, 23, 24, 27]
        J = self.constraint_jacobian()
        J[:, 0:6] = 0
        Jd = J[:, ind + dep]
        Jd[Jd < 1e-5] = 0
        M = self.full_mass_matrix()[np.ix_(ind + dep, ind + dep)]
        G = np.linalg.lstsq(Jd[:, 16:], -Jd[:, :16], rcond=None)[0]
        P = np.vstack([np.eye(16), G])
        return P.T @ M @ P

    def check_self_collision(self):
        return bool(self.L.cassie_sim_check_self_collision(self.c))

    def check_obstacle_collision(self):
        return bool(self.L.cassie_sim_check_obstacle_collision(self.c))

    def __del__(self):
        try:
            if getattr(self, 'c', None):
                self.L.cassie_sim_free(self.c)
                self.c = None
        except Exception:
            pass


# ---------------------------------------------------------------- multi-GPU: environments are independent, shard them by index
def env_shard(n_total, rank, world):
    """contiguous env-index range [start, start+count) owned by `rank` (SURVEY.md section 8e): sizes differ by at most one."""
    base, rem = divmod(int(n_total), int(world))
    count = base + (1 if rank < rem else 0)
    start = rank * base + min(rank, rem)
    return start, count


def gather_observations(local_obs, group=None):
    """the one optional collective of the path: all-gather of every rank's [n_local, OBS_WIDTH] observation block
    (torch.distributed: NCCL over NVLink on GPUs, gloo in the CPU tests).  Ranks may own different env counts."""
    import torch
    import torch.distributed as dist
    world = dist.get_world_size(group)
    counts = [torch.zeros(1, dtype=torch.int64, device=local_obs.device) for _ in range(world)]
    dist.all_gather(counts, torch.tensor([local_obs.shape[0]], dtype=torch.int64, device=local_obs.device), group=group)
    counts = [int(c.item()) for c in counts]
    if len(set(counts)) == 1:
        out = torch.empty((world * counts[0],) + tuple(local_obs.shape[1:]), dtype=local_obs.dtype, device=local_obs.device)
        dist.all_gather_into_tensor(out, local_obs.contiguous(), group=group)
        return out
    mx = max(counts)
    pad = torch.zeros((mx,) + tuple(local_obs.shape[1:]), dtype=local_obs.dtype, device=local_obs.device)
    pad[:local_obs.shape[0]] = local_obs
    parts = [torch.empty_like(pad) for _ in range(world)]
    dist.all_gather(parts, pad, group=group)
    return torch.cat([p[:c] for p, c in zip(parts, counts)], dim=0)
