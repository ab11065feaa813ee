// devmodel.h -- the per-model constant block the stepper reads (one copy per CTA in shared memory, staged with a
// TMA bulk copy), the HBM state layout, and the per-warp scratch layout.  Shared by the CUDA build (kernels.cu) and
// by the test-only host emulation of the same source (tests/emu/).
#pragma once
#include <cstdint>
#ifdef __CUDACC__
#define CASSIE_HD __host__ __device__
#else
#define CASSIE_HD
#endif

namespace cassie {

constexpr int MB = 32;        // bodies (nbody <= 32: one lane per body)
constexpr int MJ = 32;        // joints
constexpr int MV = 32;        // dofs   (nv <= 32: one lane per dof)
constexpr int MG = 16;        // collision geoms on moving bodies (world pose recomputed every step)
constexpr int MGS = 16;       // static collision geoms (world body or bodies welded to it: floor plane, height field, the 15 stair boxes of cassie.xml): device ids MG .. MG + MGS - 1
constexpr int MGT = MG + MGS;
constexpr int MPAIR = 160;    // candidate geom pairs in MuJoCo's order (cassie.xml: 9 floor + 9 x 15 box + 9 leg-leg = 153), 32 per collision pass
constexpr int NPC = 8;        // distinct contact-parameter records among the pairs (mj_contactParam results)
constexpr int ME = 4;         // connect equalities
constexpr int MU = 10;        // motors
constexpr int NM_MAX = 320;   // sparse mass-matrix entries (307 for Cassie)
constexpr int NTRI_MAX = 276; // off-diagonal entries of the sparse factor (275 for Cassie)
constexpr int NFAC_MAX = 1520; // rank-1 update pairs of the factorisation schedule (1519 for Cassie)
constexpr int NEFC = 48;      // constraint rows per env (12 equality + limits + 4 per floor contact); excess contacts are dropped and counted
constexpr int MAXCON = 12;    // contacts per env
constexpr int YSTRIDE_MAIN = 33;  // row stride of the constraint matrix in shared memory: dofs + 1 (odd: bank-conflict free both ways)
constexpr int YSTRIDE_MAX = 39;   // with the 6 dofs of an extra free body (cassie_tray_box.xml)

// model features a kernel instance is compiled for (template parameter FEAT): an instance without a feature carries none of its code
constexpr int F_XB = 1, F_HFIELD = 2, F_BOX = 4, F_ALL = 7;   // extra free body (cassie_tray_box.xml's cup), height field, box geoms
constexpr int F_EG = 8;   // the static geoms' world poses, sizes and bounding radii come from per-environment rows (GEOM_ENV_W) instead of the model block
constexpr int F_FR = 16;  // frame rows (FRAME_W per named body / site) are filled in the last sub-step of a launch (extended instances only)
constexpr int F_TR = 32;  // per-environment terrain: the bank entry from a selection row, the height field's size from its F_EG slot (with F_ALL | F_EG only)
constexpr int F_BP = 64;  // per-environment body offsets: each body's position in its parent frame comes from a BP_W row instead of the model block (extended instances only)
constexpr int F_AC = 128; // per-environment actuators: ctrlrange, no-load speed and torque delay of every motor come from an ACT_W row (with F_BP, extended instances only)
constexpr int F_MC = 256; // per-environment mechanics: link inertia, rotor armature and hinge springs come from a MECH_W row (with F_BP | F_AC, extended instances only)
constexpr int F_CT = 512; // per-environment contact softness: each contact row mixes solref / solimp from its geoms' CONTACT_W slots (with F_BP | F_AC | F_MC, extended only)
constexpr int F_XF = 1024; // per-environment applied forces: xfrc_applied / qfrc_applied from an APPLIED_W row (plain F_BOX twins, and extended with F_BP | F_AC | F_MC | F_CT)
constexpr int F_TC = 2048; // per-tick trace: every tick of a step launch stores the traced columns into a TRACE row slot (the F_XF chain twins' twins only)
constexpr int F_CL = 4096; // contact lists: the last sub-step of a step / forward launch stores its contacts into a CON_W row (the F_FR chain twins' twins only)
constexpr int F_SN = 8192; // sensor models: encoder offsets and noise, IMU mount, bias and noise from an SN_W row, drawn every tick (the F_XF twins' twins only)

CASSIE_HD inline int pair_g1(uint32_t c) { return (int)(c & 63u); }
CASSIE_HD inline int pair_g2(uint32_t c) { return (int)((c >> 6) & 63u); }
CASSIE_HD inline int pair_kind(uint32_t c) { return (int)((c >> 12) & 15u); }
CASSIE_HD inline int pair_pc(uint32_t c) { return (int)((c >> 16) & 15u); }
CASSIE_HD inline int pair_rank(uint32_t c) { return (int)((c >> 20) & 255u); }

// pair kinds handled by the narrow phase
enum PairKind { PAIR_PLANE_SPHERE = 0, PAIR_PLANE_CAPSULE = 1, PAIR_CAPSULE_CAPSULE = 2, PAIR_HFIELD_SPHERE = 3, PAIR_HFIELD_CAPSULE = 4,
                PAIR_PLANE_BOX = 5, PAIR_SPHERE_BOX = 6, PAIR_CAPSULE_BOX = 7, PAIR_BOX_BOX = 8 };

template <typename real>
struct DevModel {
  // ---- sizes / options
  int qpos_w, qvel_w, ystride, xb;   // HBM row widths, constraint-matrix row stride, id of the extra free body (or -1)
  int xb_qadr, xb_dadr, xb_jnt, any_jnt_pos;   // any_jnt_pos: some joint anchor is not at its body origin
  int nq, nv, nbody, njnt, ngeom, npair, neq, nu, maxdepth, nM, ntri, nsub, iterations, imu_body, has_damping, force_zpath;
  real timestep, tolerance, pgs_scale, root_mass_inv, euler_eps, padr[3];
  real gravity[3], magnetic[3], imu_pos[3], imu_quat[4], imu_mat[9], gyro_cutoff, accel_cutoff;
  int hf_nrow, hf_ncol, padh[2];
  real hf_size[4];           // height field: x half-size, y half-size, elevation scale, base thickness
  real xb_mass, xb_inertia[3], xb_dsqi[6], padxb[2];  // extra free body: mass, principal inertia (inertial frame = body frame), 1/sqrt of its diagonal mass matrix
  // ---- bodies
  int body_parent[MB], body_depth[MB], body_jntadr[MB], body_jntnum[MB], body_lastdof[MB], body_subtree_end[MB];
  uint32_t body_kid_dofs[MB];   // bodies with a large subtree: (first dof + 1) of up to 4 direct children, 8 bits each, 0 = none; their subtree sums are composed from the children's (0: summed directly)
  int any_big, padb[3];
  uint32_t body_dofmask[MB];
  real body_pos[MB][3], body_quat[MB][4], body_ipos[MB][3], body_imat[MB][9], body_mass[MB], body_inertia[MB][3], body_invw[MB];
  // mirror symmetry of the dof tree (two identical legs below a common base chain): lets the row transform and the A = Y Y' products skip the
  // leg a constraint row does not touch.  body_side: 0 base / world / extra body, 1 first leg, 2 second leg
  int sym_on, sym_first, sym_n, sym_madr;
  int spec19, padsp[3];   // the dof tree is the one csrc/cassie_tree_gen.inc was generated for: single-leg rows take the straight-line transform
  unsigned char body_side[MB];
  // ---- joints
  int jnt_type[MJ], jnt_qposadr[MJ], jnt_dofadr[MJ], jnt_body[MJ], jnt_limited[MJ];
  real jnt_pos[MJ][3], jnt_axis[MJ][3], jnt_stiffness[MJ], jnt_range[MJ][2], jnt_qpos0[MJ], jnt_qspring[MJ], jnt_solref[MJ][2], jnt_solimp[MJ][5];
  // ---- dofs
  int dof_body[MV], dof_jnt[MV], dof_parent[MV], dof_Madr[MV], dof_depth[MV], dof_cvelsrc[MV], dof_Mrow[MV], dof_subtree_end[MV];
  unsigned char dof_anc[MV][16];  // t-th ancestor of a dof (t = 1: parent)
  uint32_t dof_ancmask[MV];
  real dof_armature[MV], dof_damping[MV], dof_invweight0[MV];
  uint32_t tri[NTRI_MAX];     // (i << 24) | (j << 16) | qLD address of L(i,j); i descending, ancestors nearest first
  int nfac, fac_start[MV + 1], padf[2];
  uint32_t fac_pairs[NFAC_MAX];  // (t << 24) | (src << 12) | dst: qLD[dst] -= qLD[src] * f_t, grouped by eliminated dof k
  // ---- collision geoms and pairs
  int geom_body[MGT], geom_type[MGT], ngeom_static, root_body, npair_a, static_box_mask, padn[2];   // npair_a: pairs without a static box come first
  real geom_pos[MG][3], geom_mat[MG][9];   // moving geoms: frame in their body (row-major rotation)
  real geom_wpose[MGS][12];                // static geoms: world pose as the collision stage wants it (position, z axis, x axis, y axis)
  real geom_size[MGT][3], geom_rbound[MGT];   // sizes, bounding-sphere radius (0: plane / height field)
  real robot_reach, padg[3];               // no robot collision geom reaches farther than this from the root body's origin (obstacle broad phase)
  // candidate pairs: (g1 | g2 << 6 | kind << 12 | parameter record << 16 | rank in MuJoCo's pair order << 20); records = distinct mj_contactParam
  // results.  Stored in two runs, each in MuJoCo's order: [0, npair_a) the pairs without a static box, [npair_a, npair) the static-box pairs, which are
  // only visited when a box is within the robot's reach; contacts are put back into MuJoCo's order by rank afterwards
  uint32_t pair_code[MPAIR];
  int pc_condim[NPC], pc_mu_src[NPC];   // mu_src: how the sliding friction follows from the geoms': 0 max of both (equal priority), 1 geom 1, 2 geom 2
  int pc_flags[NPC];    // derived-quantity flags: bit 0 obstacle geom involved (geom user == 1), bit 1 robot-robot (both user == 2),
                        // bits 8.. : geom groups g met by a group-1 geom (cassie_sim_geom_collision, src/cassiemujoco.c:1944-1961)
  real pc_mu[NPC], pc_margin[NPC], pc_gap[NPC], pc_solref[NPC][2], pc_solimp[NPC][5];
  real qpos0[44];       // the reference configuration (mj_setConst works there)
  // ---- feet (src/cassiemujoco.c:861-866): body ids, toe / heel points in the foot frames, total mass including the extra free body
  int foot_body[2], padfb[2];
  real toe_local[2][3], heel_local[2][3], foot_offset, total_mass_inv, padft[2];
  // ---- equality
  int eq_b1[ME], eq_b2[ME];
  real eq_data[ME][6], eq_solref[ME][2], eq_solimp[ME][5];
  // ---- motors and encoders (model/cassie.xml:258-287)
  int act_dof[MU], act_qposadr[MU], enc_bits[16], enc_qposadr[16], pad2[2];
  real act_gear[MU], act_ctrl_lo[MU], act_ctrl_hi[MU], act_wmax[MU], act_torque_limit[MU], enc_scale[16];
};

// ---- HBM state: one row per environment in each array (row-major, env index slowest)
constexpr int QPOS_W_MAIN = 36, QVEL_W_MAIN = 32;   // row widths for the nq 35 / nv 32 models (runtime values live in DevModel::qpos_w / qvel_w)
constexpr int QPOS_W_XB = 44, QVEL_W_XB = 40;       // with an extra free body (nq 42 / nv 38)
constexpr int CST_W = 192;      // controller / sensor state, layout below
constexpr int DFILT_W = 96;     // int32 drive FIR taps [10][9], then DF_TICK
constexpr int DF_TICK = 90;     // control ticks since the last reset (int32): the clock of the optional open-loop gait generator
constexpr int GAIT_W = 24;      // optional per-env sinusoidal gait on the motor-PD targets: amplitude[10], phase[10], frequency (Hz), pad
constexpr int GA_AMP = 0, GA_PHASE = 10, GA_FREQ = 20;
constexpr int PD_W = 52;        // torque, pTarget, dTarget, pGain, dGain for the 10 motors (+2 pad)
constexpr int TASK_W = 64;      // optional task-space PD rows: per leg torque, pTarget, dTarget, pGain, dGain [6] each (left 0..29, right 30..59)
constexpr int XFRC_W = 8;       // force xyz, torque xyz, body id (as real), pad
constexpr int OBS_W = 112;      // the dynamic subset of cassie_out_t copied out at src/cassiemujoco.c:1127 + the decoded estimator outputs (stateless part, then the filtered part)
// CST offsets
constexpr int CS_SENSOR = 0;    // sensordata[29]
constexpr int CS_ACTVEL = 32;   // actuator_velocity[10]
constexpr int CS_DPOS = 42, CS_DVEL = 52, CS_DTORQUE = 62;   // cassie_out drive position / velocity / torque
constexpr int CS_JPOS = 72, CS_JVEL = 78;                    // cassie_out joint position / velocity
constexpr int CS_DELAY = 84;    // torque_delay[10][6]
constexpr int CS_JFX = 144;     // joint filter x[6][4]
constexpr int CS_JFY = 168;     // joint filter y[6][3]
constexpr int CS_TIME = 186;
constexpr int CS_STO = 187;     // radio channel 8 (safe-torque-off when < 1)
// OBS offsets
constexpr int OB_MPOS = 0, OB_MVEL = 10, OB_MTORQUE = 20, OB_JPOS = 30, OB_JVEL = 36, OB_QUAT = 42, OB_GYRO = 46, OB_ACCEL = 49, OB_MAG = 52, OB_TIME = 55;
// stateless part of the reference's estimator (state_output_step, closed source; semantics recovered by probing the archive, DESIGN.md):
constexpr int OB_EST_ACC = 56;    // [3] pelvis.translationalAcceleration
constexpr int OB_FOOT = 60;       // [2][13] per foot: position 3, orientation 4 (pelvis frame), rotational velocity 3, translational velocity 3 (foot frame)
constexpr int OB_EST_QUAT = 86;   // [4] pelvis.orientation (IMU quaternion through its rotation matrix and back: +-q)

// derived-quantity row (optional, cassie_batch_enable_aux): the reference's read-only queries (src/cassiemujoco.c:1586-1961) as by-products
// in-kernel estimator (optional, extended instance): per environment a row of doubles with the filter state (doubles in every precision: the
// covariance recursion is the reference's unsymmetrised one and needs them) and a row of reals with its outputs
constexpr int EST_W = 128;      // doubles: [0] started, [1..42] x axis (state 6, covariance 36), [43..84] y axis, [85..89] z state, [90..114] z covariance,
constexpr int ES_X = 1, ES_Z = 85, ES_PZ = 90, ES_TERRAIN = 115, ES_FORCE = 116;   // [115] terrain, [116..121] leg forces (toeForce of each foot, double)
constexpr int OB_EST_OUT = 96;  // [EO_W] the estimator's force model and filters, columns of the observation row (zero until cassie_batch_enable_estimator_device)
constexpr int EO_W = 16;        // reals: pelvis.position 3, translationalVelocity 3, externalForce 3, terrain.height 1, toeForce (= heelForce) L 3, R 3
constexpr int EO_POS = 0, EO_VEL = 3, EO_EXTF = 6, EO_TERRAIN = 9, EO_TOE = 10;
constexpr int AUX_W = 64;
constexpr int AX_FOOT_FORCE = 0;                    // [12] cassie_sim_foot_forces: left xyz, 3 zeros, right xyz, 3 zeros
constexpr int AX_TOE_FORCE = 12, AX_HEEL_FORCE = 18; // [6] [6] cassie_sim_heeltoe_forces: left xyz, right xyz
constexpr int AX_FOOT_POS = 24;                     // [6]  cassie_sim_foot_positions
constexpr int AX_FOOT_VEL = 30;                     // [12] cassie_sim_foot_velocities
constexpr int AX_CM_POS = 42, AX_CM_VEL = 45, AX_ANGMOM = 48;   // [3] each: centre of mass, its velocity, angular momentum about it
constexpr int AX_OBSTACLE = 51, AX_SELF = 52, AX_GROUPMASK = 53, AX_NCON = 54;
constexpr int AX_TMP = 56;                          // [8] toe / heel world xy of both feet, carried between stages of one sub-step

// per-environment model constants (optional, domain randomisation: src/cassiemujoco.c:1303-1436 setters + mj_setConst :949-977).
// When a batch carries these rows the step kernel reads the listed constants from the env's row instead of the shared model block.
constexpr int CE_W = 288;
constexpr int CE_MASS = 0;       // [32] body_mass
constexpr int CE_IPOS = 32;      // [32][3] body_ipos
constexpr int CE_DAMP = 128;     // [32] dof_damping (main tree)
constexpr int CE_FRIC = 160;     // [32] sliding friction per collision geom (device geom ids: moving 0..15, static 16..31)
constexpr int CE_BINVW = 192;    // [32] body_invweight0 (translational)  -- written by the set_const launch
constexpr int CE_DINVW = 224;    // [32] dof_invweight0                    -- written by the set_const launch
constexpr int CE_ROOT_MINV = 256, CE_TOT_MINV = 257, CE_PGS_SCALE = 258;   // 1 / main-tree mass, 1 / total mass, 1 / (meaninertia * nv)

// per-environment placement of the static collision geoms (optional, terrain curricula: stairs / tilted floors that differ between environments).
// Slot k describes device geom MG + k in the layout the collision stage reads: world pose [12] (position, z, x, y axes, as DevModel::geom_wpose), size [3],
// bounding radius [1].  A model input like the CE rows: snapshots and resets leave it alone.
constexpr int GE_SLOT = 16;
constexpr int GEOM_ENV_W = MGS * GE_SLOT;
constexpr int GE_POSE = 0, GE_SIZE = 12, GE_RBOUND = 15;
// per-environment terrain (optional, cassie_batch_set_env_hfield; F_TR instances): environment e stands on bank entry (unsigned)terrain[e] % K, and the
// height field's slot of its F_EG row holds its position (GE_POSE, the model's axes) and its x / y half-extents and elevation scale (GE_SIZE); the base
// thickness is kept on the host only.  Without a selection row the slot's size is not read and the model block's hf_size applies.
// per-environment body offsets (optional, cassie_batch_set_env_body_pos; F_BP instances): MuJoCo's body_pos of every body [MB][3] in model body order,
// the rest of the row zero.  The kinematics, the ray and the camera kernels read it instead of DevModel::body_pos.  A model input like the CE rows.
constexpr int BP_W = MB * 3;
// per-environment actuators (optional, cassie_batch_set_env_actuators; F_AC instances): per motor i MuJoCo's actuator_ctrlrange (lo, hi) -- the
// ctrllimited clamp of the actuation and motor()'s tmax --, the no-load speed wmax = actuator_user * 2 pi / 60 (rad/s) and the torque delay in control
// ticks, stored as a real; the kernel reads it clamped to [0, 6] (NaN: 0) and truncated.  A model input like the CE rows.
constexpr int ACT_W = 40;
constexpr int AC_LO = 0, AC_HI = 10, AC_WMAX = 20, AC_DELAY = 30;
constexpr int AC_MAXDELAY = 6;   // the length of the delay line (cst CS_DELAY [10][6]): the reference's TORQUE_DELAY_CYCLES
// per-environment mechanics (optional, cassie_batch_set_env_mechanics; F_MC instances): MuJoCo's body_inertia (principal moments) of every body [MB][3] in
// model body order, and per main-tree dof its dof_armature and the jnt_stiffness / qpos_spring of its joint; entries past nbody / nv zero.  The cinert
// phase reads the inertia, the CRB phase the armature (the diagonal of M and of M + hB), the passive force the spring of a hinge dof only: slide, ball
// and free joints keep the model block's (the pelvis slides carry cassie_sim_hold's spring).  A model input like the CE rows.
constexpr int MECH_W = 192;
constexpr int MC_INERTIA = 0, MC_ARMATURE = 96, MC_STIFF = 128, MC_SPRING = 160;
// per-environment contact softness (optional, cassie_batch_set_env_contact; F_CT instances): slot k describes device geom k (moving 0..15, static 16..31,
// the numbering of CE_FRIC) with MuJoCo's geom_solref [2], geom_solimp [5] and geom_solmix [1].  The constraint stage mixes each contact row's pair from
// the two slots by mj_contactParam's rule (the record's priority, else solmix); condim, margin, gap and friction stay the record's / CE_FRIC's.  Slots
// without a collision geom are zero and never read.  A model input like the CE rows.
constexpr int CT_SLOT = 8;
constexpr int CONTACT_W = MGT * CT_SLOT;
constexpr int CT_SOLREF = 0, CT_SOLIMP = 2, CT_SOLMIX = 7;
// per-environment applied forces (optional, cassie_batch_set_applied_forces; F_XF instances): MuJoCo's xfrc_applied of every body [MB][6] in model body
// order (force xyz, torque xyz in the world frame, at the body's centre of mass xipos), then qfrc_applied per dof column (main tree 0..31, the extra free
// body 32..37, as the DYN columns).  State like qvel: resets zero it, snapshots carry it.  The XFRC slot keeps its meaning and adds to its body's entry.
constexpr int APPLIED_W = 232;
constexpr int AP_XFRC = 0, AP_QFRC = 192;
// per-tick trace (optional, cassie_batch_set_trace; F_TC instances): per environment a row [T][k] of reals, slot s = what the traced columns held after
// tick s of the last step launch (its last T ticks when it ran more).  Column c of the trace is described by the batch's table entry
// (source << TC_SHIFT) | column; the sources below.  An output like the aux row: resets and snapshots leave it alone, only step launches write it.
constexpr int TC_QPOS = 0, TC_QVEL = 1, TC_OBS = 2, TC_AUX = 3, TC_FRAME = 4, TC_NSRC = 5;
constexpr int TC_SHIFT = 16, TC_COLMASK = 0xffff;
constexpr int TRACE_MAX = 64;   // columns
// contact lists (optional, cassie_batch_enable_contacts; F_CL instances): per environment MuJoCo's d->contact and mj_contactForce of the last sub-step of a
// step or forward launch (the state that sub-step started from, as the reference's queries read them after mj_step, src/cassiemujoco.c:1586-1606,
// 1781-1898): a header of CON_HEAD reals -- contacts listed (those that entered the solve, in MuJoCo's order), contacts the collision stage found,
// contacts dropped at the capacities (found - listed), zeros -- then MAXCON slots of CON_SLOT reals.  Slot: geom1, geom2 in the model's numbering, condim,
// dist, pos [3], frame [9] (row 0 the normal from geom1 to geom2, rows 1 and 2 the tangents), the contact-frame force [6] (normal, two tangential, three
// torques that are zero at condim <= 3), the friction the pyramid used, the contact's first constraint row; unused slots are zero with geoms -1.  An
// output like the aux row: resets, set_state and snapshots leave it alone.  Both widths are multiples of 16 bytes in either precision.
constexpr int CON_HEAD = 8, CON_SLOT = 24, CON_W = CON_HEAD + MAXCON * CON_SLOT;
constexpr int CN_GEOM1 = 0, CN_GEOM2 = 1, CN_DIM = 2, CN_DIST = 3, CN_POS = 4, CN_FRAME = 7, CN_FORCE = 16, CN_MU = 22, CN_EFC = 23;
static_assert(CON_W == 296 && CON_HEAD % 4 == 0 && CON_SLOT % 4 == 0, "contact-list row layout");
// sensor models (optional, cassie_batch_set_env_sensors; F_SN instances): per environment the offset and noise std of the 16 encoders in cassie_out order
// (10 drives, then 6 joints; output radians), the IMU mount quaternion (w x y z, applied as q (x) q_m), and the orientation noise std (rad, a small rotation
// on the right), the gyro bias and noise std, the accelerometer bias and noise std.  A model input like the CE rows.  The generator rows [n][SR_W] are int32:
// the Philox key (seed lo, hi) and the tick counter (lo, hi), which step launches advance by their tick count; resets and snapshots leave both alone.
constexpr int SN_W = 52;
constexpr int SN_ENC_OFF = 0, SN_ENC_STD = 16, SN_QUAT = 32, SN_ORI_STD = 36, SN_GYRO_BIAS = 39, SN_GYRO_STD = 42, SN_ACC_BIAS = 45, SN_ACC_STD = 48;
constexpr int SN_NCH = 25;   // noise channels: 16 encoders, orientation 3, gyro 3, accelerometer 3 (channel c: word c % 4 of Philox block c / 4)
constexpr int SR_W = 4;

// frames (optional, cassie_batch_set_frames): per environment a row [count][FRAME_W] describing named bodies / sites as the reference's queries see them
// after mj_step / mj_forward (src/cassiemujoco.c:1242-1252, 1543-1553, 1752-1809): poses of the state the last sub-step started from, velocities and
// contact forces of that sub-step.  Site slots carry zero velocity and force.
constexpr int FRAME_W = 20;
constexpr int FR_POS = 0, FR_QUAT = 3, FR_VEL = 7, FR_CFRC = 13;   // [3] xpos / site_xpos, [4] xquat / mat2quat(site_xmat), [6] cvel, [6] contact force (3..5 zero)
constexpr int FRAME_MAX = 64;
// the batch's frame table (global memory, one per batch): per frame body id, kind (0 body, 1 site), the site's position and orientation in its body frame
constexpr int FT_W = 12;
constexpr int FT_BODY = 0, FT_KIND = 1, FT_POS = 2, FT_QUAT = 5;
// Jacobian of one frame at the current state (launch mode 4, cassie_batch_frame_jacobian): per environment [6][FJ_COLS], rows jacp x y z then jacr x y z,
// column = dof in the reference's order (main tree 0..31, the extra free body 32..37), unused columns zero
constexpr int FJ_COLS = 40;
constexpr int FRAME_JAC_W = 6 * FJ_COLS;
// dynamics at the current state (launch mode 5, cassie_batch_dynamics): per environment the dense mass matrix (mj_fullM of qM, armature included), the
// bias forces qfrc_bias, the 3 neq rows of the connect equalities (efc_J's first rows, j1 - j2) and their p1 - p2 (efc_pos), and the offset of the
// centre of mass from the pelvis at identity pelvis orientation (cassie_sim_centroid_inertia).  Column = dof in the reference's order (main tree 0..31,
// the extra free body 32..37), unused entries zero; the row is padded to a multiple of 32
constexpr int DY_COLS = 40, DY_EQ_ROWS = 3 * ME;
constexpr int DY_M = 0, DY_BIAS = DY_M + DY_COLS * DY_COLS, DY_JEQ = DY_BIAS + DY_COLS, DY_EQPOS = DY_JEQ + DY_EQ_ROWS * DY_COLS, DY_RCM = DY_EQPOS + DY_EQ_ROWS;
constexpr int DYN_W = (DY_RCM + 3 + 31) / 32 * 32;
// inverse dynamics at the current state and a caller's qacc (launch mode 6, cassie_batch_inverse; mj_inverse of MuJoCo 2.1.0): per environment
// qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint and qfrc_constraint = J' f of the constraint rows at that qacc, column = dof as in the
// dynamics row, then the row count, the contacts with rows and the contacts dropped at the capacities, as reals; the row is padded to a multiple of 32.
// The caller's qacc comes from the batch's inverse-input rows [n][qvel width], which the launch passes as its warm start
constexpr int IV_COLS = 40;
constexpr int IV_QFRC = 0, IV_QFRCC = IV_QFRC + IV_COLS, IV_NEFC = IV_QFRCC + IV_COLS, IV_NCON = IV_NEFC + 1, IV_DROPPED = IV_NCON + 1;
constexpr int INV_W = (IV_DROPPED + 1 + 31) / 32 * 32;
// accelerations (optional, cassie_batch_enable_accelerations): per environment a row [ACC_W(count)] filled in the last sub-step of a step or forward
// launch (F_FR instances): the constraint-solved qacc (cassie_sim_qacc, src/cassiemujoco.c:1216-1219; column = dof as in the dynamics row, zeros beyond
// nv), then per frame of the batch's frame list cacc after mj_comVel + mj_rnePostConstraint (cassie_sim_body_acceleration, :1762-1771) in com-based
// coordinates (angular 3, linear 3) and 2 pad.  Site slots read zero; a body without dofs reads its parent's cacc.
constexpr int AC_QCOLS = 40, AC_SLOT = 8;
constexpr int AC_QACC = 0, AC_CACC = AC_QCOLS;
CASSIE_HD inline constexpr int acc_width(int nframes) { return AC_QCOLS + AC_SLOT * nframes; }

// ---- per-warp scratch (in units of `real`)
constexpr int S_XPOS = 0;                       // [32][3]
constexpr int S_XQUAT = S_XPOS + 96;            // [32][4]
constexpr int S_XMAT = S_XQUAT + 128;           // [32][9]
constexpr int S_CDOF = S_XMAT + 288;            // [32][6]
constexpr int S_QLD = S_CDOF + 192;             // [320] (qM itself lives in a global scratch row)
constexpr int S_DINV = S_QLD + NM_MAX;          // [32]
constexpr int S_DSQI = S_DINV + 32;             // [32]
constexpr int S_QPOS = S_DSQI + 32;             // [44]
constexpr int S_VEC = S_QPOS + 44;              // [6][32] general vectors ([96..127]: IMU stash; [128..159]: exchange buffer; [160..183]: extra-body qvel / qacc_smooth / qacc_ws / qacc (F_FR instances, for the acceleration row); [184..186]: centre of mass)
constexpr int S_CON = S_VEC + 192;              // [MAXCON][16]
constexpr int S_EFC = S_CON + MAXCON * 16;               // [NEFC][4]: row-build scalars {.., pos, src, ineq} then solver constants {b, 1/A, A, +-R}
constexpr int S_Y = S_EFC + 4 * NEFC;           // [NEFC][ystride] constraint matrix; before the constraint stage it holds the temporaries below
CASSIE_HD inline constexpr int scratch_reals(int ystride) { return S_Y + NEFC * ystride; }
// the extended instance (derived-quantity rows) appends a [32][6] copy of cdof that outlives the constraint stage
CASSIE_HD inline constexpr int scratch_reals_ext(int ystride) { return scratch_reals(ystride) + 192; }
// temporaries inside the S_Y region (dead before the first constraint row is written)
constexpr int T_CINERT = 0;                     // [32][10]
constexpr int T_CRB = 320;                      // [32][10]; during kinematics: xanchor[32][3], xaxis[32][3], qloc[32][4]; later chain sums [32][6]
constexpr int T_CVEL = 640;                     // [32][6]
constexpr int T_CFRC = 832;                     // [32][6]
constexpr int T_CDOFD = 1024;                   // [32][6]
constexpr int T_GEOM = 1216;                    // [16][12] geom world poses (position + rotation by columns), live from the collision stage until the contact list is written
constexpr int T_CBUF = 0;                       // [4 x 7][32] collision: the contacts of each lane's candidate pair, [pos3 normal3 dist] each, lane index fastest
constexpr int T_CSORT = 0;                      // [MAXCON][16] after the collision passes: the unsorted contact list while it is put back into MuJoCo's order
static_assert(T_GEOM + 192 <= NEFC * YSTRIDE_MAIN, "temporaries must fit in the constraint-matrix region");
static_assert(T_CBUF + 28 * 32 <= T_GEOM && T_CSORT + 16 * MAXCON <= T_GEOM, "the collision buffers must not overlap the geom poses");
static_assert(NEFC >= 48 && 16 * YSTRIDE_MAX <= S_QLD - S_XPOS, "the dense solver path keeps A in rows 32..47 of Y and in the kinematics buffers");
// slots of a row's 4 scalars while the rows are being built (overwritten by the solver constants afterwards)
constexpr int E_POS = 0, E_SRC = 1, E_INEQ = 2, E_SIDE = 3;   // E_SIDE: 0 / 1 the row touches the base and at most the first leg, 2 ... the second leg, 3 both legs


// ---- debug dump (tests only; one block per env, in `real`)
constexpr int D_XPOS = 0, D_XQUAT = 96, D_CDOF = 224, D_QM = 416, D_QLD = 736, D_BIAS = 1056, D_PASSIVE = 1088, D_SMOOTH = 1120,
              D_QACCS = 1152, D_QACC = 1184, D_QFRCC = 1216, D_COUNTS = 1248, D_EFC_B = 1252, D_EFC_F = 1316, D_EFC_R = 1380,
              D_EFC_AREF = 1444, D_SENS = 1508, D_J = 1540, D_SIZE = 3600;

}  // namespace cassie
