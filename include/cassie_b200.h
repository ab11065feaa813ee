/* cassie_b200.h -- C-ABI of the H100-native (sm_90a) batched Cassie stepper (libcassie_b200.so).
 *
 * Drop-in boundary for ONE path of osudrl/cassie-mujoco-sim: cassie_sim_step_pd and the few lifecycle / state verbs a caller
 * needs around it.  Every entry point cites the reference interface it replaces (paths relative to the original project).
 * Plain pointers and sizes only; no CUDA or torch types appear in any signature (device pointers travel as void*).
 *
 * Two groups:
 *   (1) legacy single-environment verbs with the reference's exact names and signatures (include/cassiemujoco.h) --
 *       a cassie_sim_t is a batch of one environment stepped by the same CUDA kernels (there is no CPU backend);
 *   (2) the new batched verbs (cassie_batch_*, cassie_sim_step_pd_batch) named by BASELINE.json's north_star.
 */
#ifndef CASSIE_B200_H
#define CASSIE_B200_H
#include <stdbool.h>
#include "cassie_bus.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct cassie_sim cassie_sim_t;     /* include/cassiemujoco.h:31 */
typedef struct cassie_state cassie_state_t; /* include/cassiemujoco.h:32 */
typedef struct cassie_batch cassie_batch_t; /* new */

/* ------------------------------------------------------------------ (1) legacy single-environment verbs */
/* include/cassiemujoco.h:45  (src/cassiemujoco.c:820-879): loads and caches the model; here: compiles the MJCF (or .cmodel) */
bool cassie_mujoco_init(const char *modelfile);
/* include/cassiemujoco.h:49  (src/cassiemujoco.c:881-...): drops the cached model */
void cassie_cleanup(void);
/* include/cassiemujoco.h:67  (src/cassiemujoco.c:979-1036): NULL on failure, message on stderr */
cassie_sim_t *cassie_sim_init(const char *modelfile, bool reinit);
/* include/cassiemujoco.h:77  (src/cassiemujoco.c:1102-1113): NULL is a no-op */
void cassie_sim_free(cassie_sim_t *sim);
/* new: the one-environment batch a simulator steps, owned by it (not to be freed), so that the batch verbs -- per-environment rows such as
 * cassie_batch_set_env_actuators or cassie_batch_set_env_mechanics, device pointers -- apply to a legacy simulator; cassie_sim_copy copies what they set. */
cassie_batch_t *cassie_sim_batch(cassie_sim_t *c);
/* include/cassiemujoco.h:95  (src/cassiemujoco.c:1147-1157): THE hot path, one environment, one 0.5 ms tick */
void cassie_sim_step_pd(cassie_sim_t *sim, state_out_t *y, const pd_in_t *u);
/* include/cassiemujoco.h:104,147,183 (src/cassiemujoco.c:1191-1214): borrowed read-write pointers (35 / 32 / 1 doubles) into a
 * host mirror; writes are uploaded before the next step, the mirror is refreshed after every step */
double *cassie_sim_time(cassie_sim_t *sim);
double *cassie_sim_qpos(cassie_sim_t *sim);
double *cassie_sim_qvel(cassie_sim_t *sim);
/* src/cassiemujoco.c:1232-1235: mjData's qfrc_applied [nv] as a borrowed read-write host mirror, uploaded before the next launch and refreshed after it
 * like cassie_sim_qpos; the first call gives the simulator's batch its applied-force rows (cassie_batch_set_applied_forces) */
double *cassie_sim_qfrc(cassie_sim_t *sim);
/* src/cassiemujoco.c:1038-1052 */
int cassie_sim_nv(const cassie_sim_t *sim);
int cassie_sim_nq(const cassie_sim_t *sim);
/* include/cassiemujoco.h:263 (src/cassiemujoco.c:1963-1967): xfrc = force xyz, torque xyz in the world frame; unknown name: no-op */
/* This verb fills ONE (wrench, body) slot per environment: a call that names another body REPLACES the earlier wrench.  For several bodies at once (the
 * reference keeps xfrc_applied per body) use the applied-force rows, cassie_batch_set_applied_forces on cassie_sim_batch(sim); the slot adds to them.
 * cassie_sim_clear_forces empties the slot and zeroes the rows' xfrc_applied.  The BASELINE configurations push the pelvis only. */
void cassie_sim_apply_force(cassie_sim_t *sim, double xfrc[6], const char *name);
/* include/cassiemujoco.h:268 (src/cassiemujoco.c:1969-1972) */
void cassie_sim_clear_forces(cassie_sim_t *sim);
/* include/cassiemujoco.h:281 (src/cassiemujoco.c:2008-2033) */
void cassie_sim_full_reset(cassie_sim_t *sim);
/* sizes the reference's Python wrapper asks for (src/cassiemujoco.c:1038-1060) and qpos += h qvel (src/cassiemujoco.c:1183-1189; *y is zeroed: the
 * reference runs its estimator on an uninitialised cassie_out_t there) */
int cassie_sim_nbody(const cassie_sim_t *sim);
int cassie_sim_ngeom(const cassie_sim_t *sim);
int cassie_sim_njnt(const cassie_sim_t *sim);
int cassie_sim_nu(const cassie_sim_t *sim);
void cassie_integrate_pos(cassie_sim_t *sim, state_out_t *y);
/* ---- the verbs RL wrappers call around the hot path
 * include/cassiemujoco.h:85 (src/cassiemujoco.c:1137-1145): user torques -> safety layer -> motor model -> physics; *y = the bus of this tick.
 * cassie_sim_step_ethercat (below the safety layer) stays a stub: the kernel always runs cassie_core_sim_step. */
void cassie_sim_step(cassie_sim_t *sim, cassie_out_t *y, const cassie_user_in_t *u);
/* src/cassiemujoco.c:1159-1181: cassie_sim_step_pd with ONE physics step per call whatever the model's timestep */
void cassie_sim_step_pd_no2khz(cassie_sim_t *sim, state_out_t *y, const pd_in_t *u);
/* src/cassiemujoco.c:2090-2092: the bus as the last step's sensors filled it (dynamic subset; the rest as cassie_out_init leaves it, :672-734) */
cassie_out_t cassie_sim_get_cassie_out(cassie_sim_t *sim);
/* include/cassiemujoco.h:108-112 (src/cassiemujoco.c:1196-1204): the physics timestep; control ticks stay 0.5 ms = round(5e-4 / timestep) sub-steps.
 * The pointer is a host mirror: a write takes effect at the next step / forward.  cassie_batch_set_timestep: the same for a batch (0 / -1). */
double *cassie_sim_timestep(cassie_sim_t *sim);
void cassie_sim_set_timestep(cassie_sim_t *sim, double dt);
int cassie_batch_set_timestep(cassie_batch_t *b, double dt);
/* src/cassiemujoco.c:1221-1225: mj_forward on the current state; returns 0 */
int cassie_sim_forward(cassie_sim_t *sim);
/* include/cassiemujoco.h:271-275 (src/cassiemujoco.c:1974-2000): pin / free the pelvis (stiff spring-damper on its slides, damping on its ball joint) */
void cassie_sim_hold(cassie_sim_t *sim);
void cassie_sim_release(cassie_sim_t *sim);
/* src/cassiemujoco.c:1466-1541 (example/test_terrain.c:118-157 builds stairs out of the 15 boxes of model/cassie.xml:232-246 with them): geom position /
 * orientation / size in the reference's geom numbering; borrowed pointers are host mirrors, a change takes effect at the next step / forward.
 * All 135 box x robot candidate pairs are collided (contact rules for boxes: DESIGN.md section 3); a box out of the robot's reach costs one
 * distance test per step.  cassie_batch_set_geom_pose: the same for a batch, one placement shared by its environments (NULL: leave that part). */
double *cassie_sim_geom_pos(cassie_sim_t *sim);
double *cassie_sim_geom_quat(cassie_sim_t *sim);
double *cassie_sim_geom_size(cassie_sim_t *sim);
double *cassie_sim_geom_name_pos(cassie_sim_t *sim, const char *name);
int cassie_sim_mj_name2id(cassie_sim_t *sim, char *mj_type, char *name);   /* cassie_batch_name2id on the sim's batch */
double *cassie_sim_geom_name_quat(cassie_sim_t *sim, const char *name);
double *cassie_sim_geom_name_size(cassie_sim_t *sim, const char *name);
void cassie_sim_set_geom_pos(cassie_sim_t *sim, double *pos);
void cassie_sim_set_geom_quat(cassie_sim_t *sim, double *quat);
void cassie_sim_set_geom_size(cassie_sim_t *sim, double *size);
void cassie_sim_set_geom_name_pos(cassie_sim_t *sim, const char *name, double *pos);
void cassie_sim_set_geom_name_quat(cassie_sim_t *sim, const char *name, double *quat);
void cassie_sim_set_geom_name_size(cassie_sim_t *sim, const char *name, double *size);
int cassie_batch_set_geom_pose(cassie_batch_t *b, const char *name, const double *pos, const double *quat, const double *size);
/* Per-environment placement of a static plane or box (src/cassiemujoco.c:1466-1541, one placement per environment): terrain curricula whose stairs
 * and floor tilt differ between the environments of a batch.  pos [n][3] / quat [n][4] are the geom's frame in its body, as MuJoCo's geom_pos /
 * geom_quat (the same meaning as in cassie_batch_set_geom_pose); size [n][3].  A NULL part leaves that part alone; mask [n] (or NULL: all) selects
 * the environments that change, the others keep theirs.  The first call gives every environment a row initialised from the shared placement; only the
 * touched geom's slot is uploaded.  Unlike the shared verb, a per-environment box's bounding radius is recomputed as |size|, so a box enlarged beyond
 * its file size is never culled by a stale bound.  The placement is part of the model, not of the state: reset and snapshot restore leave it alone.
 * cassie_batch_set_geom_pose while rows exist still means one placement for all: it also rewrites that geom's slot in every row.
 * 0, or -1 with nothing changed (cassie_b200_last_error) for an unknown geom, a geom on a moving body, the height field, or a geom without a
 * collision slot.  get: the placement each environment sees [n][3] / [n][4] / [n][3] (any part may be NULL), rows or not.  clear: frees the rows,
 * the batch follows the shared placement again. */
int cassie_batch_set_env_geom_pose(cassie_batch_t *b, const char *name, const double *pos, const double *quat, const double *size, const unsigned char *mask);
int cassie_batch_get_env_geom_pose(cassie_batch_t *b, const char *name, double *pos, double *quat, double *size);
int cassie_batch_clear_env_geom_poses(cassie_batch_t *b);

/* Frames: named bodies and sites of the model ("world" included) whose state every step / forward launch writes as a by-product, for rewards and
 * observations built from the robot's own frames.  Per environment a row [count][CASSIE_FRAME_WIDTH] in the batch precision (environment slowest);
 * per frame, what the reference's queries return after cassie_sim_step_pd / cassie_sim_forward (src/cassiemujoco.c:1242-1252, 1543-1553,
 * 1752-1809):
 *   CASSIE_FRAME_POS  [3] body: xpos; site: site_xpos                               } of the state the last physics sub-step started from
 *   CASSIE_FRAME_QUAT [4] body: xquat; site: mju_mat2Quat(site_xmat)                }
 *   CASSIE_FRAME_VEL  [6] body: cvel (cassie_sim_body_velocities: com-based [angular; linear], the new qvel with that sub-step's cdof); site: 0
 *   CASSIE_FRAME_CFRC [6] body: cassie_sim_body_contact_force (world force of the contacts touching the body, -/+ for body 1 / 2; slots 3..5
 *                         zero, as in the reference); site: 0
 * set: names[count] with kinds[count] (CASSIE_FRAME_BODY / CASSIE_FRAME_SITE), at most CASSIE_FRAME_MAX; the rows start at zero and are filled from the
 * next launch on.  count = 0 frees the rows.  0, or -1 with nothing changed (cassie_b200_last_error) for an unknown name or kind or too many frames.
 * get: synchronous host copy [n][count][CASSIE_FRAME_WIDTH] doubles; device pointer: cassie_batch_device_ptr(b, "frames").  Every successful set
 * reallocates the rows: a device pointer (or zero-copy view) taken before it is no longer valid.  Snapshots carry the rows and restore them into a batch
 * with the same frame list. */
#define CASSIE_FRAME_WIDTH 20
#define CASSIE_FRAME_POS 0
#define CASSIE_FRAME_QUAT 3
#define CASSIE_FRAME_VEL 7
#define CASSIE_FRAME_CFRC 13
#define CASSIE_FRAME_MAX 64
#define CASSIE_FRAME_BODY 0
#define CASSIE_FRAME_SITE 1
int cassie_batch_set_frames(cassie_batch_t *b, const char *const *names, const int *kinds, int count);
int cassie_batch_nframes(const cassie_batch_t *b);
int cassie_batch_get_frames(cassie_batch_t *b, double *out);
/* The Jacobian of frame `frame` (0 .. count-1) at the CURRENT state of every environment, as the reference's cassie_sim_get_jacobian_full(_site)
 * (src/cassiemujoco.c:1254-1301: kinematics and centre of mass recomputed, then mj_jacBody at xpos or mj_jacSite): jacp, jacr [n][3][nv] (nv = 32,
 * or 38 with the extra free body; jacr may be NULL).  One launch, synchronous; it writes nothing else (the frame rows keep the last step's poses).
 * Device rows: cassie_batch_device_ptr(b, "frame_jac") [n][6][CASSIE_FRAME_JAC_COLS] (jacp x y z, jacr x y z; column = dof, unused columns zero),
 * allocated by the first call.  0, or -1 (cassie_b200_last_error) for a frame out of range. */
#define CASSIE_FRAME_JAC_COLS 40
#define CASSIE_FRAME_JAC_WIDTH 240
int cassie_batch_frame_jacobian(cassie_batch_t *b, int frame, double *jacp, double *jacr);
/* Dynamics at the CURRENT state of every environment, for model-based controllers (operational-space control, whole-body QPs, inverse dynamics):
 * the joint-space mass matrix M(q) (mj_fullM of qM, armature included), the bias forces qfrc_bias(q, qdot) (Coriolis, centrifugal, gravity), and
 * Cassie's closed-chain constraints, the Jacobian and position error of the connect equalities (efc_J / efc_pos's first 3 neq rows), with each
 * environment's own masses and inertial offsets (cassie_batch_set_body_mass / _ipos).  The extra free body's block of M is its constant
 * diag(m, m, m, I1, I2, I3), its bias [-m g; w x I w] (translation in the world frame, rotation in the body frame).
 * cassie_batch_dynamics: one launch on the batch stream (asynchronous, like cassie_batch_query); it writes nothing else (state, observations, aux,
 * frame rows, counters).  The rows are allocated by the first call, freed with the batch; snapshots and resets leave them alone.
 * cassie_batch_get_dynamics: synchronous copy of what the last dynamics launch wrote: M [n][nv][nv], bias [n][nv], J_eq [n][3 neq][nv],
 * eq_err [n][3 neq], Icm [n][9] (cassie_sim_centroid_inertia's formula, see below); any pointer may be NULL.  -1 (cassie_b200_last_error) before
 * any dynamics launch.  Device rows: cassie_batch_device_ptr(b, "dyn") [n][CASSIE_DYN_WIDTH] in the batch precision, column = dof (main tree
 * 0..31, the extra free body 32..37), unused entries zero:
 *   CASSIE_DYN_M     [40][40] dense symmetric M
 *   CASSIE_DYN_BIAS  [40]     qfrc_bias
 *   CASSIE_DYN_JEQ   [12][40] connect rows j1 - j2, in equality order
 *   CASSIE_DYN_EQPOS [12]     their p1 - p2
 *   CASSIE_DYN_RCM   [3]      the subtree com of the world body with the pelvis turned to the identity, minus the pelvis position */
#define CASSIE_DYN_COLS 40
#define CASSIE_DYN_M 0
#define CASSIE_DYN_BIAS 1600
#define CASSIE_DYN_JEQ 1640
#define CASSIE_DYN_EQPOS 2120
#define CASSIE_DYN_RCM 2132
#define CASSIE_DYN_WIDTH 2144
int cassie_batch_dynamics(cassie_batch_t *b);
int cassie_batch_get_dynamics(cassie_batch_t *b, double *M, double *bias, double *J_eq, double *eq_err, double *Icm);
int cassie_batch_neq(const cassie_batch_t *b);
/* Inverse dynamics at the CURRENT state of every environment and a caller's joint acceleration, as MuJoCo 2.1.0's mj_inverse (continuous time): the
 * generalised force that produces qacc there, for torque labels of reference motions, system identification from logs, holding torques and forward /
 * inverse consistency checks.  With the constraint rows of the state (connect equalities, joint limits, contacts with the environment's own softness,
 * friction and terrain; the forward's capacities of 48 rows and 12 contacts) evaluated at that qacc, as mj_constraintUpdate does:
 *   jar = J qacc - aref;  f = -jar / R on equality rows; on limit and contact rows f = -jar / R if jar < 0, else 0;  qfrc_constraint = J' f
 *   qfrc_inverse = M qacc + qfrc_bias - qfrc_passive - qfrc_constraint   (M with the armature; passive: damping and springs)
 * Applied forces (xfrc_applied, qfrc_applied, the XFRC slot) and actuation are not subtracted: they are part of what qfrc_inverse returns, as in MuJoCo.
 * At the qacc of the acceleration rows (the continuous-time one, before mj_Euler's implicit-damping correction) it gives back the forward's actuator
 * and applied forces, to solver accuracy.  The extra free body's block is diag(m, m, m, I1, I2, I3) qacc + [-m g; w x I w] minus its constraint
 * columns.  Every per-environment row of the model is honoured (masses, inertial offsets, damping, body offsets, inertia, armature, springs, contact
 * softness, static geoms, terrain).
 * cassie_batch_inverse: qacc [n][nv] (host) is uploaded into the inverse-input rows, then one launch on the batch stream (asynchronous).  qacc NULL:
 * the inverse-input rows as the caller left them, for example copied on the device from the acceleration rows; after the first call that path
 * synchronises, copies and allocates nothing.  It writes nothing else (state, warm start, observations, aux, frame and acceleration rows, counters).
 * 0, or -1 (cassie_b200_last_error): NULL before the input rows exist.
 * cassie_batch_get_inverse: synchronous copy of what the last inverse launch wrote: qfrc_inverse [n][nv], qfrc_constraint [n][nv], counts [n][3] (rows,
 * contacts with rows, contacts dropped at the capacities: a lying-flat environment can be discarded); any pointer may be NULL.  -1 before any inverse
 * launch.  Device rows, in the batch precision, allocated (zero) by the first call or device-pointer request, freed with the batch, left alone by
 * snapshots and resets:
 *   cassie_batch_device_ptr(b, "inv_qacc") [n][cassie_batch_row_width(b, "qvel")]  the input: column = dof (main tree 0..31, the extra free body 32..37)
 *   cassie_batch_device_ptr(b, "inv")      [n][CASSIE_INV_WIDTH]                    the output, column = dof as in the dynamics row, unused entries zero:
 *   CASSIE_INV_QFRC    [40]  qfrc_inverse
 *   CASSIE_INV_QFRCC   [40]  qfrc_constraint
 *   CASSIE_INV_NEFC, CASSIE_INV_NCON, CASSIE_INV_DROPPED  [1] each: the counts, as reals */
#define CASSIE_INV_COLS 40
#define CASSIE_INV_QFRC 0
#define CASSIE_INV_QFRCC 40
#define CASSIE_INV_NEFC 80
#define CASSIE_INV_NCON 81
#define CASSIE_INV_DROPPED 82
#define CASSIE_INV_WIDTH 96
int cassie_batch_inverse(cassie_batch_t *b, const double *qacc);
int cassie_batch_get_inverse(cassie_batch_t *b, double *qfrc_inverse, double *qfrc_constraint, int *counts);
/* Accelerations, as step / forward by-products (joint-acceleration penalties, impact rewards, IMU-like observations at any body, acceleration-level
 * controllers): per environment a row [CASSIE_ACC_WIDTH(count)] in the batch precision, count = cassie_batch_nframes, filled in the last physics sub-step
 * of every step and forward launch (also the forward of cassie_batch_reset):
 *   CASSIE_ACC_QACC [40]  qacc (cassie_sim_qacc): the constraint-solved acceleration of that sub-step -- after a step the value the warm start keeps,
 *                         before mj_Euler's implicit-damping correction; after a forward the solved qacc, warm start untouched.  Column = dof (main
 *                         tree 0..31, the extra free body 32..37), zeros beyond nv
 *   CASSIE_ACC_CACC + CASSIE_ACC_SLOT f  [6] per frame f of the frame list: body: cacc (cassie_sim_body_acceleration: mj_comVel + mj_rnePostConstraint
 *                         on the state the step left -- the new qvel, that sub-step's cdof, its qacc -- com-based [angular; linear], gravity included as
 *                         cacc(world) = (0, 0, 0, -g)); a body without dofs reads its parent's; site: 0.  Then 2 pad
 * cassie_batch_enable_accelerations: on = 1 allocates the rows (zero until the next step or forward), 0 drops them; 0 / -1.  A batch with rows runs the
 * extended frame instance of the step kernel.  cassie_batch_set_frames reallocates them to the new width, zeroed.  Snapshots carry them and restore
 * them into a batch with the same frame list and rows.
 * cassie_batch_get_accelerations: synchronous copy, qacc [n][nv], cacc [n][count][6]; either may be NULL; -1 (error recorded, nothing copied) without
 * rows.  Device rows: cassie_batch_device_ptr(b, "acc"), width cassie_batch_row_width(b, "acc"). */
#define CASSIE_ACC_QACC 0
#define CASSIE_ACC_QCOLS 40
#define CASSIE_ACC_CACC 40
#define CASSIE_ACC_SLOT 8
#define CASSIE_ACC_WIDTH(count) (40 + 8 * (count))
int cassie_batch_enable_accelerations(cassie_batch_t *b, int on);
int cassie_batch_get_accelerations(cassie_batch_t *b, double *qacc, double *cacc);
/* Terrain sensing: rays cast against each environment's STATIC collision geoms (floor plane, height field, boxes, with the environment's own placement
 * and terrain) at the CURRENT qpos -- height scans around the pelvis for terrain curricula, and the reference's rangefinders
 * (cassie_sim_read_rangefinder below; mj_ray).  Moving geoms (the robot's own, the extra free body) are not seen.
 * cassie_batch_set_rays: k rays (0 .. CASSIE_RAY_MAX; 0 drops the table), ray i from origin[3 i] along dir[3 i] (normalised here) up to max_dist[i],
 * in frame[i]:
 *   CASSIE_RAY_HEADING  the root body's position and yaw (the yaw of its x axis on the world xy plane): turns with the heading, stays level
 *   CASSIE_RAY_ROOT     the root body's pose
 *   CASSIE_RAY_WORLD    world coordinates, the same for every environment
 * 0, or -1 with nothing changed (cassie_b200_last_error) for an unknown frame kind, a zero direction, max_dist <= 0 or k out of range.  Every
 * successful set drops the rows: a device pointer taken before it is no longer valid.
 * cassie_batch_raycast: one launch on the batch stream (asynchronous) that casts every ray of every environment; it writes nothing but the rows
 * [n][k][CASSIE_RAY_SLOT] in the batch precision (allocated by the first cast; snapshots, resets and cassie_sim_copy leave them alone):
 *   distance to the first hit (-1: none within max_dist), world z of the hit (of the ray's end point when none), static geom slot 0..15 (-1), 0
 * cassie_batch_get_rays: synchronous copy [n][k][CASSIE_RAY_SLOT] doubles; -1 before the first cast after a set.  Device rows:
 * cassie_batch_device_ptr(b, "rays"), row width k CASSIE_RAY_SLOT. */
#define CASSIE_RAY_MAX 1024
#define CASSIE_RAY_SLOT 4
#define CASSIE_RAY_HEADING 0
#define CASSIE_RAY_ROOT 1
#define CASSIE_RAY_WORLD 2
int cassie_batch_set_rays(cassie_batch_t *b, const int *frame, const double *origin, const double *dir, const double *max_dist, int k);
int cassie_batch_nrays(const cassie_batch_t *b);
int cassie_batch_raycast(cassie_batch_t *b);
int cassie_batch_get_rays(cassie_batch_t *b, double *out);
/* Depth cameras: a set of up to CASSIE_CAM_MAX cameras per batch, each mounted on a body, rendered at the CURRENT qpos of every environment as depth
 * images -- the perception signal of the reference's CassieVis draw_depth (an offscreen OpenGL render, one environment at a time), here one kernel
 * launch for the batch and every camera of the set (the body poses are composed once per environment for all of them).
 * A camera looks along its -z axis, +y is image up, fovy is the full vertical angle (degrees).  Pixel (r, c) of a width x height image is taken at
 * its centre, row 0 at the TOP; its value is the z-depth (distance along the optical axis, metres) of the first hit in (0, zfar], and zfar where
 * nothing is hit within zfar.  (The reference's mjr_readPixels buffer is bottom row first and holds OpenGL's non-linear depth; the values here are
 * linear metres.)  What is seen: the static collision geoms with the ray rules (each environment's own placement and terrain), and the moving
 * collision geoms -- the robot's spheres and capsules, boxes on moving bodies, the extra free body -- from outside only: a pixel whose ray starts
 * inside a moving geom does not see that geom.  Visual meshes are not loaded, so the robot appears as its collision model.
 * cassie_batch_set_camera: a <camera> of the model by name; only fixed-mode cameras (not the track cameras).  cassie_batch_set_camera_mount: a
 * camera the caller mounts on a named body, pos / quat in the body frame (quat is normalised).  Either returns 0, or -1 with nothing changed
 * (cassie_b200_last_error) for an unknown camera or body (the message lists the model's cameras), a camera that is not fixed, fovy outside
 * (0, 180), width or height outside 1 .. CASSIE_CAM_MAXDIM, zfar <= 0 or not finite, a zero or non-finite quaternion.  width = 0 drops the
 * camera.  Either is a set of one camera.  Every successful set drops the depth, geom-id and per-environment mount rows: a device pointer taken
 * before it is no longer valid.
 * cassie_batch_set_cameras: k cameras sharing one image size and zfar; body [k] in the model's numbering (cassie_batch_name2id(b, "body", ..)),
 * pos [k][3], quat [k][4] (normalised), fovy [k].  Each is checked as set_camera_mount checks its mount; a refusal returns -1 with nothing changed
 * and names the camera ("camera i: ...").  k = 0 drops the set.  cassie_batch_model_camera: the mount of a fixed <camera> of the model (body,
 * pos, quat as the model has them, fovy); -1 for an unknown or non-fixed camera.  cassie_batch_ncameras: k of the current set (0: none).
 * cassie_batch_render_depth: one launch on the batch stream (asynchronous); it writes nothing but the rows [n][k][height][width] in the batch
 * precision, and the geom-id rows when enabled (allocated by the first render after a set; snapshots, resets and cassie_sim_copy leave them alone).
 * cassie_batch_get_depth: synchronous copy [n][k][height][width] doubles; -1 before the first render after a set.  Device rows:
 * cassie_batch_device_ptr(b, "depth"), row width k x height x width (for k = 1 the layout of a one-camera batch).
 * Per-environment mounts (extrinsics and field-of-view randomisation): cassie_batch_set_env_cameras gives environment e's camera c its own pose in
 * the camera's body frame and its own fovy: pos [n][k][3], quat [n][k][4], fovy [n][k]; any part may be NULL (kept); mask [n] (NULL: all)
 * selects the environments that change.  The first call starts every environment from the set's mounts.  A non-finite value, a zero quaternion or
 * a fovy outside (0, 180) returns -1 with nothing changed; the error names the environment, the camera and the field.  get reports what every
 * environment sees, with or without rows; clear returns to the set's mounts.  Device rows: cassie_batch_device_ptr(b, "camera_env")
 * [n][k][CASSIE_CAMENV_SLOT] in the batch precision: pos[3], quat[4], fovy in degrees, read at the next render.  The kernel normalises the
 * quaternion and forms tan(fovy / 2) itself, so rows written on the device need no host call; a slot with a non-finite value, a zero quaternion or a
 * fovy outside (0, 180) renders nothing (zfar and geom -1 on every pixel of that camera).  The rows are a model input: resets, reset_where,
 * set_state and snapshot restores leave them alone, cassie_sim_copy copies them (between sets of as many cameras; otherwise it drops the
 * destination's).  The body of each camera is the set's in every environment.
 * Geom ids: cassie_batch_enable_camera_geoms(b, 1) makes every render also write int32 rows [n][k][height][width]
 * (cassie_batch_device_ptr(b, "camera_geom")): the model geom id (cassie_batch_id2name(b, "geom", id)) of the surface that set the pixel's depth,
 * -1 where nothing lies within zfar; on a tie the static geom, then the lower device index.  0 frees them.  cassie_batch_get_camera_geoms copies
 * them; -1 before the first render with geom ids after a set or an enable. */
#define CASSIE_CAM_MAXDIM 256
#define CASSIE_CAM_MAX 4
#define CASSIE_CAMENV_SLOT 8
int cassie_batch_set_camera(cassie_batch_t *b, const char *camera, int width, int height, double zfar);
int cassie_batch_set_camera_mount(cassie_batch_t *b, const char *body, const double pos[3], const double quat[4], double fovy,
                                  int width, int height, double zfar);
int cassie_batch_set_cameras(cassie_batch_t *b, int k, const int *body, const double *pos, const double *quat, const double *fovy, int width, int height,
                             double zfar);
int cassie_batch_model_camera(cassie_batch_t *b, const char *camera, int *body, double pos[3], double quat[4], double *fovy);
int cassie_batch_ncameras(const cassie_batch_t *b);
int cassie_batch_render_depth(cassie_batch_t *b);
int cassie_batch_get_depth(cassie_batch_t *b, double *out);
int cassie_batch_set_env_cameras(cassie_batch_t *b, const double *pos, const double *quat, const double *fovy, const unsigned char *mask);
int cassie_batch_get_env_cameras(cassie_batch_t *b, double *pos, double *quat, double *fovy);
int cassie_batch_clear_env_cameras(cassie_batch_t *b);
int cassie_batch_enable_camera_geoms(cassie_batch_t *b, int on);
int cassie_batch_get_camera_geoms(cassie_batch_t *b, int *out);
/* include/cassiemujoco.h:61-73 (src/cassiemujoco.c:1072-1093): model (per-environment constants, height field, timestep) + full dynamic state */
cassie_sim_t *cassie_sim_duplicate(const cassie_sim_t *src);
void cassie_sim_copy(cassie_sim_t *dst, const cassie_sim_t *src);
/* include/cassiemujoco.h:434-463 (src/cassiemujoco.c:3380-3452): full dynamic state of a simulator -- qpos, qvel, warm start, time, sensor snapshot,
 * cassie_out subset, encoder filters, torque delay line, applied forces, estimator filters, last observation row.  The borrowed time / qpos / qvel
 * pointers are host mirrors: what the caller writes there after cassie_get_state is honoured by cassie_set_state.  A state owns its (device)
 * memory: it can be restored into any simulator of the same model and freed at any time, before or after the simulator it was taken from. */
cassie_state_t *cassie_state_alloc(void);
cassie_state_t *cassie_state_duplicate(const cassie_state_t *src);
void cassie_state_copy(cassie_state_t *dst, const cassie_state_t *src);
void cassie_state_free(cassie_state_t *state);
double *cassie_state_time(cassie_state_t *state);
double *cassie_state_qpos(cassie_state_t *state);
double *cassie_state_qvel(cassie_state_t *state);
void cassie_get_state(const cassie_sim_t *sim, cassie_state_t *state);
void cassie_set_state(cassie_sim_t *sim, const cassie_state_t *state);
/* Import compatibility: the library also exports, as stubs, the 133 further names example/cassiemujoco_ctypes.py resolves at import time
 * (cassie_vis_*, UDP, pack / unpack, pd_input_* / cassie_core_sim_* / state_output_* host objects, mjModel / mjData accessors, ...;
 * csrc/legacy_stubs.inc, list in tests/golden/ctypes_bound_names.txt).  They are outside the accelerated path: a call records an error
 * (cassie_b200_last_error), prints it and returns 0 / NULL.  They are deliberately not declared here. */
/* include/cassiemujoco.h:317-329 (src/cassiemujoco.c:2050-2080): height-field terrain of cassie_hfield.xml; nrow*ncol floats in [0,1],
 * row-major, row <-> y, column <-> x.  cassie_sim_hfielddata returns a borrowed read-write host mirror uploaded before the next step. */
int cassie_sim_get_hfield_nrow(cassie_sim_t *sim);
int cassie_sim_get_hfield_ncol(cassie_sim_t *sim);
int cassie_sim_get_nhfielddata(cassie_sim_t *sim);
float *cassie_sim_hfielddata(cassie_sim_t *sim);
void cassie_sim_set_hfielddata(cassie_sim_t *sim, float *data);
/* the height field's size [4] (src/cassiemujoco.c:2062-2070): get returns a borrowed read-write host mirror, set copies into it; it is uploaded before
 * the next step or forward.  An invalid size is not uploaded: the error is recorded and the last valid size stays.  Without a height field: NULL / no
 * change, and an error. */
double *cassie_sim_get_hfield_size(cassie_sim_t *sim);
void cassie_sim_set_hfield_size(cassie_sim_t *sim, double size[4]);
/* read-only derived quantities (SURVEY.md 8f-2).  include/cassiemujoco.h:200-240 (src/cassiemujoco.c:1586-1699, 1812-1898, 1944-1961).
 * Like the reference, the contact / foot group reads what the LAST step left behind (contact list and forces of the state that step
 * started from); the centre-of-mass group first recomputes the kinematics of the current state (the reference calls mj_fwdPosition).
 * cm_velocity / angular_momentum use velocities consistent with that state (the reference mixes them with the previous step's cvel). */
bool cassie_sim_check_obstacle_collision(const cassie_sim_t *sim);
bool cassie_sim_check_self_collision(const cassie_sim_t *sim);
void cassie_sim_foot_forces(const cassie_sim_t *c, double cfrc[12]);
void cassie_sim_heeltoe_forces(const cassie_sim_t *c, double toe_force[6], double heel_force[6]);
bool cassie_sim_geom_collision(const cassie_sim_t *c, int geom_group);
void cassie_sim_foot_positions(const cassie_sim_t *c, double cpos[6]);   /* src/cassiemujoco.c:1608-1621 (defined there, not in the header) */
void cassie_sim_foot_velocities(const cassie_sim_t *c, double cvel[12]);
void cassie_sim_cm_position(const cassie_sim_t *c, double cm_pos[3]);
void cassie_sim_cm_velocity(const cassie_sim_t *c, double cm_vel[3]);
void cassie_sim_angular_momentum(const cassie_sim_t *c, double Lcm[3]);
/* frames of the simulator (every body and site, cassie_batch_set_frames): poses, cvel and contact forces the last step / forward left behind; host
 * mirrors laid out like mjData's xpos / xquat / site_xpos, refreshed after every step, forward and state restore.  The Jacobians run a query launch
 * at the current state.  An unknown name gives NULL / zeros and records an error.  src/cassiemujoco.c:1242-1301, 1543-1562, 1752-1809 */
double *cassie_sim_xpos(cassie_sim_t *c, const char *name);
double *cassie_sim_xquat(cassie_sim_t *c, const char *name);
double *cassie_sim_site_xpos(cassie_sim_t *c, const char *name);
void cassie_sim_site_xquat(cassie_sim_t *c, const char *name, double *xquat);
void cassie_sim_body_velocities(const cassie_sim_t *c, double cvel[6], const char *name);
void cassie_sim_body_contact_force(const cassie_sim_t *c, double cfrc[6], const char *name);
void cassie_sim_get_jacobian(cassie_sim_t *c, double *jac, const char *name);
void cassie_sim_get_jacobian_full(cassie_sim_t *c, double *jac, double *jac_rot, const char *name);
void cassie_sim_get_jacobian_full_site(cassie_sim_t *c, double *jac, double *jac_rot, const char *name);
void cassie_sim_relative_pose(double pos1[3], double quat1[4], double pos2[3], double quat2[4], double pos2_in_pos1[3], double quat2_in_quat1[4]);
/* accelerations of the simulator (src/cassiemujoco.c:1216-1219, 1762-1779), from its acceleration row: what the last step / forward left behind, like
 * cassie_sim_body_velocities.  cassie_sim_qacc: borrowed nv-entry host mirror.  cassie_sim_body_acceleration: cacc of the body (com-based [angular;
 * linear]); an unknown name gives zeros and records an error.  cassie_sim_foot_orient: the right-foot-middle site quaternion, as cassie_sim_site_xquat
 * gives it; zeros and an error for a model without that site.  cassie_sim_full_reset zeroes qacc and sets every body to (0, 0, 0, -g). */
double *cassie_sim_qacc(cassie_sim_t *c);
void cassie_sim_body_acceleration(const cassie_sim_t *c, double accel[6], const char *name);
void cassie_sim_foot_orient(const cassie_sim_t *c, double corient[4]);
/* dynamics of the simulator at its current state (src/cassiemujoco.c:1647-1749), one dynamics launch each, then host arithmetic: the 32 x 32 main-tree
 * block of M; its rows / columns {0..8, 12, 18..21, 25, 31}; the 3 + 3 rows (32 columns) of the connects whose body1 is left- / right-achilles-rod
 * and their errors (zeros and an error recorded when the model has none); and the reference's centroid inertia, m = M[0][0], I_p = M[3:6, 3:6],
 * diagonal I_p - m (r_j^2 + r_k^2), off-diagonals I_p[i][j] - m r_i r_j (the reference's sign), r = the centre of mass at identity pelvis orientation
 * minus the pelvis position.  The reference's mj_fwdPosition also rewrites d->xpos & co.; the frame mirrors keep the last step's poses. */
void cassie_sim_full_mass_matrix(const cassie_sim_t *c, double M[1024]);
void cassie_sim_minimal_mass_matrix(const cassie_sim_t *c, double M[256]);
void cassie_sim_loop_constraint_info(const cassie_sim_t *c, double J_cl[192], double err_cl[6]);
void cassie_sim_centroid_inertia(const cassie_sim_t *c, double Icm[9]);
/* the six rangefinders (src/cassiemujoco.c:776-778; example/cassiemujoco.py:175-181 sense_ground): model rangefinder i (<rangefinder site= cutoff=>,
 * recorded apart from the 29-number sensor table) casts from its site along the site's z axis, at the site poses of the mirrors (the state the last
 * physics sub-step started from, when MuJoCo evaluates the sensor), as one CASSIE_RAY_WORLD cast on the simulator's batch of one; the distance to the
 * static terrain, min(cutoff, d) where cutoff > 0, -1 for no hit; no noise, as in the reference.  Slots past the model's rangefinders read 0; a model
 * without rangefinders gets zeros and a recorded error. */
void cassie_sim_read_rangefinder(cassie_sim_t *c, double ranges[6]);
/* model constants for domain randomisation (SURVEY.md 8f-3).  src/cassiemujoco.c:1303-1436, 949-977 (most are defined there without a header
 * declaration; example/cassiemujoco.py:517-610 calls them).  The pointer-returning verbs hand out borrowed read-write host mirrors
 * ([nv], [nbody], [3 nbody], [3 ngeom] doubles, numbered like the reference's mjModel incl. its visual mesh geoms); writes are uploaded
 * before the next step / query / set_const.  What the stepper uses: dof_damping of the 32 robot dofs, body_mass, body_ipos (not of the
 * free `cup_box` body), the sliding coefficient geom_friction[3 g] of colliding geoms.  As in MuJoCo, a changed mass acts at once while
 * the solver's reference weights (body/dof_invweight0, meaninertia, subtree masses) stay stale until (just_)set_const. */
void cassie_sim_params(cassie_sim_t *c, int *params);                 /* :1566-1574: nq nv nu nsensordata nbody ngeom */
double *cassie_sim_dof_damping(cassie_sim_t *c);                       /* :1303 */
double *cassie_sim_body_mass(cassie_sim_t *c);                         /* :1308 */
double *cassie_sim_body_ipos(cassie_sim_t *c);                         /* :1313 */
double *cassie_sim_geom_friction(cassie_sim_t *c);                     /* :1318 */
void cassie_sim_set_dof_damping(cassie_sim_t *c, double *damp);        /* :1330 */
void cassie_sim_set_dof_name_damping(cassie_sim_t *c, const char *name, double *damp);   /* :1338 */
double *cassie_sim_get_dof_name_damping(cassie_sim_t *c, const char *name);              /* :1347 */
int cassie_sim_get_joint_num_dof(cassie_sim_t *c, const char *name);                     /* :1353 */
void cassie_sim_set_body_mass(cassie_sim_t *c, double *mass);          /* :1366 */
void cassie_sim_set_body_name_mass(cassie_sim_t *c, const char *name, double mass);      /* :1373 */
double cassie_sim_get_body_name_mass(cassie_sim_t *c, const char *name);                 /* :1379 */
void cassie_sim_set_body_ipos(cassie_sim_t *c, double *ipos);          /* :1385 (reads ipos[i + j], as the reference does) */
void cassie_sim_set_body_name_ipos(cassie_sim_t *c, const char *name, double *ipos);     /* :1394 */
double *cassie_sim_get_body_name_ipos(cassie_sim_t *c, const char *name);                /* :1402 */
/* src/cassiemujoco.c:1408-1418: a body's position in its parent frame (MuJoCo's body_pos).  get returns a borrowed read-write pointer into an
 * [nbody][3] host mirror, set copies 3 values into it; when the mirror changed, the constant block is rebuilt from it before the next launch (the
 * static geoms' world poses and the broad phase's robot bound follow, so moving "floor" moves the height field).  Any body is accepted; the world
 * body's and the extra free body's entries have no effect, as in MuJoCo.  The constants of mj_setConst are not refreshed: call cassie_sim_set_const.
 * An unknown name: NULL / no change, and an error (the reference indexes -1). */
void cassie_sim_set_body_name_pos(cassie_sim_t *c, const char *name, double *data);
double *cassie_sim_get_body_name_pos(cassie_sim_t *c, const char *name);
/* src/cassiemujoco.c:2114-2192: the torque delay line [10][6], the joint filters x [6][4] / y [6][3] and the drive filters [10][9], read and written
 * through the simulator's batch.  cassie_sim_joint_filter / cassie_sim_drive_filter lend host mirrors laid out as joint_filter_t[6] {double x[4], y[3]}
 * and drive_filter_t[10] {int x[9]} (the C structs; the reference's ctypes file declares double x[9] for the latter); a write through them is
 * uploaded before the next launch, like the other borrowed pointers. */
void cassie_sim_torque_delay(cassie_sim_t *c, double *t);
void cassie_sim_set_torque_delay(cassie_sim_t *c, double *t);
void cassie_sim_get_joint_filter(cassie_sim_t *c, double *x, double *y);
void cassie_sim_set_joint_filter(cassie_sim_t *c, double *x, double *y);
void cassie_sim_get_drive_filter(cassie_sim_t *c, int *x);
void cassie_sim_set_drive_filter(cassie_sim_t *c, int *x);
void *cassie_sim_joint_filter(cassie_sim_t *c);
void *cassie_sim_drive_filter(cassie_sim_t *c);
/* :1237: mjData's ctrl [nu] as the last physics step applied it (the drive torque over the gear: exact to 1 ulp).  Writes through the pointer have
 * no effect on the next step, as in the reference, where cassie_motor_data overwrites d->ctrl before mj_step; zeros after cassie_sim_full_reset
 * (:2024) until the next step. */
double *cassie_sim_ctrl(cassie_sim_t *c);
void cassie_sim_set_geom_friction(cassie_sim_t *c, double *fric);      /* :1420 */
void cassie_sim_set_geom_name_friction(cassie_sim_t *c, const char *name, double *fric); /* :1427 (addresses the geom's own triple) */
double *cassie_sim_get_geom_name_friction(cassie_sim_t *c, const char *name);            /* :1433 */
void cassie_sim_set_const(cassie_sim_t *c);                            /* :949-972: mj_setConst, then qpos <- init, qvel <- 0, time <- 0, mj_forward */
void cassie_sim_just_set_const(cassie_sim_t *c);                       /* :974-977: mj_setConst only */
/* src/cassiemujoco.c:2002-2006: the 16 radio channels; channel 8 < 1 engages safe-torque-off */
void cassie_sim_radio(cassie_sim_t *sim, double channels[16]);

/* ------------------------------------------------------------------ (2) batched verbs (new; north_star) */
#define CASSIE_B200_FP32 0 /* throughput build: state and arithmetic in fp32 */
#define CASSIE_B200_FP64 1 /* parity build: state and arithmetic in fp64 */
#define CASSIE_PD_WIDTH 52  /* compact motor-PD row: torque[10] pTarget[10] dTarget[10] pGain[10] dGain[10] pad[2] */
#define CASSIE_OBS_WIDTH 112 /* compact observation row, see cassie_batch_get_obs */
#define CASSIE_AUX_WIDTH 64 /* derived-quantity row, see cassie_batch_get_aux */
/* offsets inside a derived-quantity row */
#define CASSIE_AUX_FOOT_FORCE 0   /* [12] cassie_sim_foot_forces layout: left xyz, 3 zeros, right xyz, 3 zeros */
#define CASSIE_AUX_TOE_FORCE 12   /* [6]  cassie_sim_heeltoe_forces toe_force: left xyz, right xyz */
#define CASSIE_AUX_HEEL_FORCE 18  /* [6]  ... heel_force */
#define CASSIE_AUX_FOOT_POS 24    /* [6]  cassie_sim_foot_positions */
#define CASSIE_AUX_FOOT_VEL 30    /* [12] cassie_sim_foot_velocities */
#define CASSIE_AUX_CM_POS 42      /* [3]  centre of mass of everything (cassie_sim_cm_position) */
#define CASSIE_AUX_CM_VEL 45      /* [3]  its velocity (cassie_sim_cm_velocity) */
#define CASSIE_AUX_ANGMOM 48      /* [3]  angular momentum about it (cassie_sim_angular_momentum) */
#define CASSIE_AUX_OBSTACLE 51    /* 1 if a contact involves an obstacle geom (cassie_sim_check_obstacle_collision) */
#define CASSIE_AUX_SELF 52        /* 1 if two robot geoms touch (cassie_sim_check_self_collision) */
#define CASSIE_AUX_GROUPMASK 53   /* bit g set: a group-1 geom touches a geom of group g (cassie_sim_geom_collision) */
#define CASSIE_AUX_NCON 54        /* contacts that entered the solve */

/* n_env environments on CUDA device `device`, all in the state cassie_sim_init leaves (src/cassiemujoco.c:979-1036).
 * modelfile: MJCF (.xml) or a compiled table (.cmodel).  NULL + stderr message on failure (no GPU, bad model, ...). */
cassie_batch_t *cassie_batch_init(const char *modelfile, int n_env, int device, int precision);
void cassie_batch_free(cassie_batch_t *b);
int cassie_batch_nenv(const cassie_batch_t *b);
int cassie_batch_nq(const cassie_batch_t *b);
int cassie_batch_nv(const cassie_batch_t *b);
/* back to the cassie_sim_init state (mask == NULL: all envs; else mask[i] != 0 selects env i) */
void cassie_batch_reset(cassie_batch_t *b, const unsigned char *mask);

/* cassie_sim_step_pd for every environment: pd_in[n_env] host AoS in, state_out[n_env] host AoS out (may be NULL).
 * Replaces n_env calls of src/cassiemujoco.c:1147-1157.  Synchronous.  state_out carries the stateless part of the reference's
 * state_output_step, decoded from the closed archive and checked equal to it to 1e-11: motor / joint position + velocity + torque,
 * pelvis.orientation (+-q, mat2quat's sign), rotationalVelocity, translationalAcceleration, both feet's position / orientation (pelvis frame) and
 * footRotationalVelocity / footTranslationalVelocity (foot frame), radio, battery; toeForce / heelForce and pelvis.position /
 * translationalVelocity / externalForce, terrain.height (the spring-force model and the filters) from the in-kernel estimator, which this call
 * switches on by itself (see cassie_batch_enable_estimator_device; ..._forces / ..._filter select the host-side checker instead).
 * externalMoment and terrain.slope are zero, as they are in the reference's output.
 * Deviation: the reference runs state_output_step in every cassie_sim_step_pd call; here the estimator comes on at the first call that passes
 * state_out, so a caller whose first k calls pass NULL gets filters that start k ticks late (as after cassie_batch_reset_estimator at that call).
 * Calls with NULL state_out before that run the kernel without the estimator stage. */
void cassie_sim_step_pd_batch(cassie_batch_t *envs, const pd_in_t *pd_in, state_out_t *state_out);

/* throughput path: compact rows.  pd: host [n_env][CASSIE_PD_WIDTH] doubles, copied to the device (and converted to the batch
 * precision) on the batch stream; step: `nticks` control ticks per launch with the PD rows held; asynchronous. */
void cassie_batch_set_pd(cassie_batch_t *b, const double *pd);
/* the taskPd branch of pd_in_t (include/pd_in_t.h:32-38) for the throughput path: host [n_env][60] doubles = per leg (left, right)
 * torque[6] pTarget[6] dTarget[6] pGain[6] dGain[6]; NULL switches the branch off.  Task coordinates as the reference's closed
 * pd_input_step uses them (decoded, pinned to the archive): foot position in the pelvis frame, then yaw / pitch / roll of the foot
 * frame; rates in the foot frame.  cassie_sim_step_pd(_batch) forward pd_in_t's taskPd fields automatically.  0 / -1. */
int cassie_batch_set_task_pd(cassie_batch_t *b, const double *rows);
/* Open-loop gait on top of the motor-PD rows (BASELINE config 5 "random PD gaits", SURVEY.md 8d): in every control tick of every launch
 * pTarget_i(t) = row.pTarget_i + amp_i sin(2 pi freq t + phase_i), t = control ticks since the last reset (or since this call) x 0.5 ms.
 * amp [n][10], freq [n] (Hz), phase [n][10]; all NULL switches it off.  New verb: the reference moves its targets from the host every tick. */
int cassie_batch_set_pd_gait(cassie_batch_t *b, const double *amp, const double *freq, const double *phase);
void cassie_batch_step(cassie_batch_t *b, int nticks);
void cassie_batch_sync(cassie_batch_t *b);
/* host copies (synchronous): qpos [n][35], qvel [n][32], time [n], obs [n][CASSIE_OBS_WIDTH] =
 * motor pos[10] vel[10] torque[10], joint pos[6] vel[6], IMU quat[4] gyro[3] accel[3] mag[3], time (0..55);
 * estimator: translationalAcceleration[3] (56), pad, per foot {position 3, orientation 4, rotational velocity 3, translational
 * velocity 3} left (60..72) right (73..85), pelvis.orientation[4] (86..89; the IMU quaternion up to sign), pad;
 * in-kernel estimator (cassie_batch_enable_estimator_device; zero while it is off): pelvis.position[3] (96), translationalVelocity[3] (99),
 * externalForce[3] (102), terrain.height (105), toeForce = heelForce left[3] (106) right[3] (109) */
void cassie_batch_get_qpos(cassie_batch_t *b, double *out);
void cassie_batch_set_qpos(cassie_batch_t *b, const double *in);
void cassie_batch_get_qvel(cassie_batch_t *b, double *out);
void cassie_batch_set_qvel(cassie_batch_t *b, const double *in);
void cassie_batch_get_time(cassie_batch_t *b, double *out);
void cassie_batch_get_obs(cassie_batch_t *b, double *out);
/* derived quantities for every environment, as by-products of the step kernel (no second pass over the state).
 * enable_aux(b, 1) allocates [n][CASSIE_AUX_WIDTH] rows in the batch precision; from then on every step / forward launch fills them:
 * contact-derived slots and foot positions / velocities exactly as the reference's queries would return right after that step; the
 * centre-of-mass slots describe the state the last sub-step STARTED from (one 0.5 ms tick old).  cassie_batch_query recomputes only the
 * centre-of-mass slots for the CURRENT state and writes nothing else (state, sensors and the other slots are untouched).
 * get_aux: synchronous host copy [n][CASSIE_AUX_WIDTH] doubles; device pointer: cassie_batch_device_ptr(b, "aux").  0 / -1. */
int cassie_batch_enable_aux(cassie_batch_t *b, int on);
int cassie_batch_get_aux(cassie_batch_t *b, double *out);
int cassie_batch_query(cassie_batch_t *b);
/* per-environment model constants (domain randomisation).  rows are host [n][width] doubles in the host model's numbering (= the
 * reference's mjModel): body_mass [nbody], body_ipos [3 nbody], dof_damping [nv], geom_friction [3 ngeom].  The first call allocates a
 * 1 KB (fp32) constant row per environment that the step kernel then reads instead of the shared model block.  set_const runs mj_setConst
 * for the selected environments (mask == NULL: all) as one kernel launch at the reference configuration -- body/dof inverse weights, subtree
 * masses, mean inertia -- and, with reset_state != 0, the state reset of cassie_sim_set_const (src/cassiemujoco.c:955-971).  0 / -1. */
int cassie_batch_nbody(const cassie_batch_t *b);
int cassie_batch_ngeom(const cassie_batch_t *b);
int cassie_batch_njnt(const cassie_batch_t *b);   /* joints of the model (the stiffness / springref width of cassie_batch_set_env_mechanics) */
int cassie_batch_set_body_mass(cassie_batch_t *b, const double *mass);
int cassie_batch_set_body_ipos(cassie_batch_t *b, const double *ipos);
int cassie_batch_set_dof_damping(cassie_batch_t *b, const double *damp);
int cassie_batch_set_geom_friction(cassie_batch_t *b, const double *fric);
int cassie_batch_get_body_mass(cassie_batch_t *b, double *mass);
int cassie_batch_get_body_ipos(cassie_batch_t *b, double *ipos);
int cassie_batch_get_dof_damping(cassie_batch_t *b, double *damp);
int cassie_batch_get_geom_friction(cassie_batch_t *b, double *fric);
int cassie_batch_set_const(cassie_batch_t *b, const unsigned char *mask, int reset_state);
/* toeForce / heelForce of state_out_t (the estimator's spring-force model, decoded; single-precision agreement with the archive): computed
 * on the host while cassie_sim_step_pd_batch unpacks its rows; off by default for batches (host time per environment), always on for a
 * cassie_sim_t.  The pure function behind it is exported for callers that keep observations on the device:
 * ang = hipRoll, hipYaw, hipPitch, knee (motor positions), shin, tarsus (joint encoders), foot (motor position); quat = IMU quaternion. */
int cassie_batch_enable_estimator_forces(cassie_batch_t *b, int on);
void cassie_b200_estimator_leg_force(int side, const double ang[7], const double quat[4], double force[3]);
/* The estimator's filters (state_output_step's stateful part, src/cassiemujoco.c:1180; decoded from the closed block's memory, agreement with the
 * archive 1e-13 on the archive's own stateless outputs): pelvis.position, translationalVelocity, externalForce, terrain.height.  One filter
 * object per environment lives on the host and advances once per cassie_sim_step_pd_batch call (the reference runs it once per 2 kHz
 * step_pd call); it turns the force option on.  Off by default for batches, always on for a cassie_sim_t.  cassie_batch_reset_estimator
 * restarts the filters (state_output_setup; mask as in cassie_batch_reset).  The filter is also exported as a plain host object:
 * ..._step reads orientation, translationalAcceleration, both feet's position and toe / heel forces from *y and writes the four outputs. */
int cassie_batch_enable_estimator_filter(cassie_batch_t *b, int on);
/* The same estimator inside the step kernel (leg forces + filters, every 2 kHz tick of a launch, so multi-tick launches keep it exact and
 * device-resident observations are complete): columns 96..111 of the observation row ("obs"), also copied out by cassie_batch_get_estimator --
 * pelvis.position 3, translationalVelocity 3, externalForce 3, terrain.height 1, toeForce (= heelForce) left 3, right 3.
 * The filter state is held in doubles in every batch precision.  cassie_batch_reset(_estimator) restarts it.
 * cassie_sim_step_pd_batch switches it on by itself at the first call that asks for state_out_t rows, because cassie_sim_step_pd runs
 * state_output_step in every call (src/cassiemujoco.c:1156); cassie_batch_enable_estimator_device(b, 0) keeps it off (the filtered fields,
 * toeForce and heelForce of state_out_t are then zero).  A cassie_sim_t always runs it. */
#define CASSIE_EST_WIDTH 16
int cassie_batch_enable_estimator_device(cassie_batch_t *b, int on);
int cassie_batch_get_estimator(cassie_batch_t *b, double *out /* [n][CASSIE_EST_WIDTH] */);
int cassie_batch_reset_estimator(cassie_batch_t *b, const unsigned char *mask);
void *cassie_b200_estimator_filter_new(void);
void cassie_b200_estimator_filter_free(void *filter);
void cassie_b200_estimator_filter_reset(void *filter);
void cassie_b200_estimator_filter_step(void *filter, state_out_t *y);
/* measurement aids: accumulated wall-clock seconds of cassie_sim_step_pd_batch since the last reset -- out[0] host pack of pd_in_t[], out[1] device part
 * (H2D, kernel, D2H, as waited for), out[2] host unpack into state_out_t[], out[3] number of calls, out[4] / out[5] milliseconds of the H2D copy /
 * of the kernel by CUDA events (only when the environment variable CASSIE_B200_AOS_EVENTS is set); CPUs this process may use (affinity mask
 * clipped by the cgroup quota), which bounds the pack / unpack threads (CASSIE_B200_AOS_THREADS, default 32) */
void cassie_batch_aos_timing(cassie_batch_t *b, double out[6], int reset);
int cassie_b200_effective_cpus(void);
/* OpenMP threads cassie_sim_step_pd_batch packs / unpacks with: CASSIE_B200_AOS_THREADS, else the CPUs above minus two (at most 32) */
int cassie_b200_aos_threads(void);
/* Batched snapshots (new): every row array of the batch copied device-to-device into an opaque handle; restore all environments or the masked
 * subset (mask as in cassie_batch_reset; e.g. return the fallen robots of an RL batch to a stored standing state).  0 / -1. */
void *cassie_batch_state_alloc(cassie_batch_t *b);
void cassie_batch_state_free(cassie_batch_t *b, void *state);
int cassie_batch_get_state(cassie_batch_t *b, void *state);
int cassie_batch_set_state(cassie_batch_t *b, const void *state, const unsigned char *mask);
/* re-run mj_forward on the current state (after set_qpos / set_qvel), like cassie_sim_forward (src/cassiemujoco.c:1221-1225) */
void cassie_batch_forward(cassie_batch_t *b);
/* Device-side resets (new): environments restored from a bank of K start states under a mask that lives on the device, with no host round trip.
 *
 * cassie_batch_set_reset_bank: entry i of the bank becomes environment envs[i] (envs NULL: i) of `state`, a snapshot taken with
 * cassie_batch_state_alloc / cassie_batch_get_state.  The snapshot may come from another batch of any size, so K may exceed n and poses prepared in a
 * helper batch (qpos / qvel written through the device pointers, cassie_batch_forward, cassie_batch_get_state) can be banked; it must have the same
 * precision and model (qpos / qvel widths) and live on the same device.  The gather runs on the device.  Every call replaces the bank; k == 0 or state
 * NULL frees it.  0, or -1 with the old bank kept for k < 0, an envs index outside the snapshot, or a snapshot of another precision or model.
 * cassie_batch_reset_bank_size: K (0 without a bank).
 *
 * cassie_batch_reset_where: environment e with d_mask[e] != 0 (device uint8[n]; a torch.bool tensor as it is) takes bank entry
 * (unsigned)d_entry[e] % K (device int32[n]; NULL: e % K), so no value can address outside the bank.  The semantics are those of
 * cassie_batch_set_state applied to the chosen entry, per environment; the rows of unmasked environments are not touched.  Optional rows: estimator
 * and applied-force rows the batch has are copied from the entry, or zeroed when the bank lacks them (the filters start afresh); aux rows are copied
 * when both have them, else left alone; frame and acceleration rows are copied when the frame lists are equal, else left alone.  A row kind the bank
 * has and the batch lacks is ignored (nothing is allocated).  counters, PD, task and gait rows and every model input are left alone; time is the
 * entry's own.  One launch, enqueued on the batch's stream: no host synchronisation, no copy, no allocation, so it can be captured in a CUDA graph.
 * The mask and entries must be written before the launch in the batch's stream order.  -1, with nothing enqueued, for: no bank, a NULL mask, a
 * pointer that is not device or managed memory of the batch's device, the host-side estimator filters on (cassie_batch_enable_estimator_filter),
 * or the batch of a cassie_sim_t (cassie_sim_batch).
 *
 * cassie_batch_forward_where: mj_forward for the environments with d_mask[e] != 0 (as cassie_batch_forward, on their own model rows), the others
 * untouched; asynchronous and capture-safe like reset_where, with its pointer checks.  Use it after writing qpos / qvel of reset environments on the
 * device (per-episode noise), or after an entry taken under other model rows, to recompute the sensor data, aux, frame and acceleration rows
 * with each environment's own model rows (the observation row follows at the next control tick, as after cassie_batch_forward).  A batch with applied-force rows gets
 * model-valued contact rows at its first extended launch, which allocates: until an ordinary cassie_batch_step or cassie_batch_forward has run,
 * forward_where refuses with -1. */
int cassie_batch_set_reset_bank(cassie_batch_t *b, const void *state, const int *envs, int k);
int cassie_batch_reset_bank_size(const cassie_batch_t *b);
int cassie_batch_reset_where(cassie_batch_t *b, const void *d_mask, const void *d_entry);
int cassie_batch_forward_where(cassie_batch_t *b, const void *d_mask);
/* Loop closure (new): each selected environment's qpos and qvel projected onto the model's connect equalities, for start states that did not come from
 * the simulator (noise on qpos, retargeted motions, poses from motor angles, body offsets inside a loop), which would otherwise start with open loops that
 * the constraint rows pull shut over the first ticks.
 *
 * Loop-closure rules that are ours:
 * - Equations: every connect equality, with MuJoCo's definition p1 = xpos[b1] + xmat[b1] eq_data[0..2], p2 = xpos[b2] + xmat[b2] eq_data[3..5], residual
 *   r = p1 - p2 (4 x 3 rows for the Cassie models).  A model without connect equalities makes the call a no-op that returns 0.
 * - Free coordinates: every main-tree joint that is not on the root body (the root body's joints -- a free joint, or the pelvis's three slides and ball
 *   -- place the tree in the world), drives no actuator and has zero jnt_stiffness in the model table.  For the Cassie models: the achilles-rod ball,
 *   tarsus, foot crank and plantar rod of each leg.  Every other coordinate (pelvis, motors including the foot, shin and heel springs, the extra free
 *   body) is held bitwise.
 * - Positions: the free ball joints' quaternions are normalised, then damped Gauss-Newton steps dq_f = -J_f' (J_f J_f' + lambda I)^-1 r run, J_f being the
 *   translational Jacobian difference of the anchor points in the free columns; a ball joint turns by its step through the step integrator's quaternion
 *   update.  They stop when max |r| <= tol or after max_iter steps.  lambda = 1e-10 m^2 in fp64, 1e-6 m^2 in fp32: the rows of a planar loop (a Cassie
 *   leg's plantar-rod loop) are rank-deficient, so J_f J_f' is singular; lambda sits above its rounding and far below its smallest non-zero eigenvalue
 *   (~1.2e-3 m^2 for Cassie).
 * - Velocities, at the closed pose: qvel_f <- qvel_f - J_f' (J_f J_f' + lambda I)^-1 (J qvel), so that J qvel ~ 0 (up to lambda / 1.2e-3 of it in the
 *   weakest direction); held velocities are unchanged.
 * - Per-environment body offsets (cassie_batch_set_env_body_pos) move the anchors and are honoured; no other per-environment row enters.
 * - An environment that is not within tol after max_iter steps keeps its qpos and qvel bitwise and reports -1 iterations; one already within tol keeps
 *   its qpos bitwise (0 iterations) and still has its velocity projected.  Unselected environments, their status rows included, are not touched.
 * - The launch writes qpos, qvel and the status rows only: follow it with cassie_batch_forward_where(mask) to refresh sensordata, aux, frames and the
 *   observation, as after cassie_batch_reset_where plus noise.
 *
 * cassie_batch_close_loops: d_mask is device uint8[n] (a torch.bool tensor as it is), NULL for every environment.  One launch on the batch's stream: no
 * host synchronisation, copy or allocation, so it can be captured in a CUDA graph -- except the first call, which allocates and zeroes the status rows
 * (make it before a capture).  -1, with nothing enqueued, for a mask that is not device or managed memory of the batch's device, max_iter outside
 * 1..CASSIE_LOOP_MAX_ITER, a tol that is not finite and > 0, a connect equality on the extra free body, or the batch of a cassie_sim_t.
 * cassie_batch_device_ptr(b, "loops"): the status rows [n][CASSIE_LOOP_SLOT] in the batch precision: the residual max |p1 - p2| after the launch (metres;
 * for a failure, that of the unchanged pose), the iterations used (0: already closed, -1: not converged), max |J qvel| after the launch, a pad.
 * cassie_batch_get_loop_status: their synchronous host copy, [n] each; any pointer may be NULL.  -1 before the first cassie_batch_close_loops. */
#define CASSIE_LOOP_SLOT 4
#define CASSIE_LOOP_MAX_ITER 200
#define CASSIE_LOOP_RESIDUAL 0
#define CASSIE_LOOP_ITERATIONS 1
#define CASSIE_LOOP_VEL_RESIDUAL 2
int cassie_batch_close_loops(cassie_batch_t *b, const void *d_mask, int max_iter, double tol);
int cassie_batch_get_loop_status(cassie_batch_t *b, double *residual, int *iterations, double *vel_residual);
/* Inverse kinematics (new): each selected environment's free coordinates posed so that up to CASSIE_IK_MAX body or site frames reach per-environment
 * position and orientation targets, for resets onto terrain, reference motions given as foot poses and task-space targets.
 *
 * Rules that are ours:
 * - Target list (per batch, shared by every environment): cassie_batch_set_ik(b, names, kinds, frames, weights, count).  kinds[i]: CASSIE_FRAME_BODY /
 *   CASSIE_FRAME_SITE; frames[i]: CASSIE_IK_WORLD, or CASSIE_IK_ROOT for a target expressed in the root body's (the pelvis's) frame (NULL: all world);
 *   weights[i][6] weight the position rows x, y, z (the expression frame's axes) and the orientation rows about the target frame's x, y, z; a weight of 0
 *   drops its row (a Cassie foot: position plus pitch and yaw -- with the position fixed the leg cannot set all three angles).  The orientation error is
 *   the rotation vector of R_target' R_frame, in the target's axes.  count 0 drops the list and its rows.  The call allocates the rows below (zero), so
 *   a solve allocates nothing.  Refused: more than CASSIE_IK_MAX targets, an unknown name or kind, a frame other than the two, a negative or non-finite
 *   weight, a target whose weights are all zero, a target on a body that no free coordinate moves (the pelvis, the extra free body), a connect equality
 *   on the extra free body, the batch of a cassie_sim_t.
 * - Free coordinates: the main-tree joints off the root body with zero jnt_stiffness -- the motors plus close_loops' free set, 22 columns for Cassie.
 *   Everything else (the root joints, the shin and heel springs at their given deflection, the extra free body) and every unselected environment is
 *   held bitwise.  The start point is the environment's qpos, which picks the branch (a knee forward); per-environment body offsets are honoured.
 * - Positions: the loops are closed with close_loops' steps (motors held), then Levenberg-Marquardt steps run on the weighted task rows with the connect
 *   rows held to first order; every limited free hinge or slide stays in its jnt_range by a projected step (a column at a bound whose step points
 *   outward is dropped for that step); after each step the loops are re-closed, motors held, to min(tol, 1e-12 m) in fp64 / min(tol, 1e-6 m) in fp32;
 *   a step is accepted only if the task residual sum (w e)^2 falls, else the damping grows tenfold and the step is retried.  The task residual thus
 *   never rises above its value at the (closed) start.  The loop re-closing moves close_loops' own joints and does not hold their ranges.
 * - Velocities (velocities = 0): the motors keep their qvel, the loops' passive joints are projected onto the loops as close_loops does.  (velocities =
 *   1): one damped least-squares fit of the free qvel at the final pose, the connect rows held exactly, so that each target frame's linear velocity and
 *   its angular velocity about the weighted axes match the target rows: world targets are world-frame velocities (the held pelvis motion included),
 *   root targets velocities relative to the pelvis in its axes.
 * - Outcome: 1 reached (position and orientation rows within tol, state written); 2 best effort (the target is out of reach or held by a range: the
 *   steps stalled or max_iter ran out; the closest pose found is written, loops closed); -1 the start pose's loops could not be closed or a NaN appeared
 *   (state kept).  The launch writes qpos, qvel and the status rows only: follow it with cassie_batch_forward_where(mask).
 * - Snapshots, cassie_sim_copy, reset_where and the per-environment row blocks do not carry the target or status rows: they are a work area.
 *
 * cassie_batch_device_ptr(b, "ik_targets"): [n][CASSIE_IK_MAX][CASSIE_IK_TARGET_WIDTH] in the batch precision, written by the caller: position (3),
 * quaternion (4, normalised on read), linear velocity (3), angular velocity (3, the expression frame's axes), pad.  "ik": the status rows
 * [n][CASSIE_IK_SLOT]: position residual (m), orientation residual (rad) -- the largest error over the weighted rows --, loop residual (m),
 * iterations, outcome, max |J_eq qvel| after the launch, velocity residual (the largest error over the weighted velocity rows; 0 for velocities = 0),
 * the number of free joints at a bound.
 * cassie_batch_solve_ik: d_mask is device uint8[n] (a torch.bool tensor as it is), NULL for every environment.  One launch on the batch's stream: no
 * host synchronisation, copy or allocation, so it can be captured in a CUDA graph.  -1, with nothing enqueued, for no target list, a mask that is not
 * device or managed memory of the batch's device, max_iter outside 1..CASSIE_IK_MAX_ITER, a tol (metres and radians) that is not finite and > 0,
 * velocities other than 0 / 1, or the batch of a cassie_sim_t.  cassie_batch_get_ik_status: the status rows' synchronous host copy [n][CASSIE_IK_SLOT]. */
#define CASSIE_IK_MAX 4
#define CASSIE_IK_TARGET_WIDTH 16
#define CASSIE_IK_SLOT 8
#define CASSIE_IK_MAX_ITER 500
#define CASSIE_IK_WORLD 0
#define CASSIE_IK_ROOT 1
#define CASSIE_IK_POS 0
#define CASSIE_IK_QUAT 3
#define CASSIE_IK_VEL 7
#define CASSIE_IK_ANGVEL 10
#define CASSIE_IK_POS_RESIDUAL 0
#define CASSIE_IK_ORI_RESIDUAL 1
#define CASSIE_IK_LOOP_RESIDUAL 2
#define CASSIE_IK_ITERATIONS 3
#define CASSIE_IK_OUTCOME 4
#define CASSIE_IK_JEQ_QVEL 5
#define CASSIE_IK_VEL_RESIDUAL 6
#define CASSIE_IK_AT_BOUND 7
int cassie_batch_set_ik(cassie_batch_t *b, const char *const *names, const int *kinds, const int *frames, const double *weights, int count);
int cassie_batch_solve_ik(cassie_batch_t *b, const void *d_mask, int max_iter, double tol, int velocities);
int cassie_batch_get_ik_status(cassie_batch_t *b, double *status);
/* batched cassie_sim_apply_force / cassie_sim_clear_forces: xfrc [n][6]; one (wrench, body) slot per env, added to the applied-force rows
 * (cassie_batch_set_applied_forces) when the batch has them; clear_forces empties the slot and zeroes the rows' xfrc_applied, keeping qfrc_applied */
int cassie_batch_apply_force(cassie_batch_t *b, const double *xfrc, const char *body_name);
void cassie_batch_clear_forces(cassie_batch_t *b);
/* batched cassie_integrate_pos (src/cassiemujoco.c:1183-1189 -> mj_integratePos): qpos <- qpos (+) h * qvel, the HBM-bound kernel */
void cassie_batch_integrate_pos(cassie_batch_t *b);

/* batched cassie_sim_set_hfielddata: `n_terrains` height fields of nrow*ncol floats; environment e stands on terrain e % n_terrains
 * (BASELINE config 4: a few dozen terrains shared round-robin).  0 on success, -1 if the model has no height field. */
int cassie_batch_set_hfielddata(cassie_batch_t *b, const float *data, int n_terrains);
int cassie_batch_hfield_nrow(const cassie_batch_t *b);
int cassie_batch_hfield_ncol(const cassie_batch_t *b);

/* Per-environment terrain (terrain curricula): which bank entry each environment stands on, and where and how large its height field is.  terrain [n]
 * (bank entry in [0, K) of cassie_batch_set_hfielddata), pos [n][3] (the height field's position in its body frame, as MuJoCo's geom_pos; it stays
 * axis-aligned), size [n][4] (x half-extent, y half-extent, elevation scale, base thickness, as hfield_size).  A NULL part leaves that part alone; mask
 * [n] (or NULL: all) selects the environments that change.  The first call gives every environment terrain e % K and the shared position and size, and
 * the batch then runs kernel instances that read them per environment.  Like the static-geom placement these are model inputs: reset and snapshot
 * restore leave them alone, cassie_sim_copy copies them.  0, or -1 with nothing changed (cassie_b200_last_error names the environment and the field)
 * when a terrain is outside [0, K), size[0] or size[1] is not > 0, size[2] or size[3] is < 0, a value is not finite, or the model has no height field.
 * get: what each environment sees (any pointer may be NULL), with or without rows.  clear: back to terrain e % K and the shared position and size.
 * The selection row is also cassie_batch_device_ptr(b, "terrain") (int32 [n], row width 1): a write there takes effect at the next launch, and
 * every kernel reads (unsigned)t % K, so no value addresses outside the bank.  cassie_batch_set_hfielddata with another K keeps the selections, which
 * are then read mod the new K.  cassie_batch_clear_env_geom_poses also returns the position and size to the shared ones and keeps the selections.
 * cassie_batch_set_hfield_size sets the shared size (the same checks; the bounding radius follows the model compiler's rule) and returns every
 * environment's position and size to the shared ones; the selections stay.  get: the shared size. */
int cassie_batch_set_env_hfield(cassie_batch_t *b, const int *terrain, const double *pos, const double *size, const unsigned char *mask);
int cassie_batch_get_env_hfield(cassie_batch_t *b, int *terrain, double *pos, double *size);
int cassie_batch_clear_env_hfield(cassie_batch_t *b);
int cassie_batch_set_hfield_size(cassie_batch_t *b, const double size[4]);
int cassie_batch_get_hfield_size(const cassie_batch_t *b, double size[4]);

/* Per-environment body offsets (domain randomisation of where a load or tray sits, and of link and mounting offsets): pos [n][nbody][3] is each
 * environment's MuJoCo body_pos (a body's position in its parent frame; body_quat stays the model's), mask [n] (or NULL: all) selects the environments
 * that change.  The first call gives every environment the model's offsets; the batch then also carries constant rows (cassie_batch_set_body_mass &
 * co.) and runs kernel instances that read the offsets per environment in the kinematics: everything that follows from the body poses (contacts,
 * sensors, connect rows, frames, Jacobians, dynamics and acceleration rows, rays, depth images) follows.  As in MuJoCo, offsets inside a leg's closed
 * loop open it at qpos0 and the connect rows pull it shut; the mj_setConst constants are not refreshed by themselves (cassie_batch_set_const); the
 * in-kernel estimator keeps the model's leg geometry.  The broad phase's robot bound is recomputed over all rows.  0, or -1 with nothing changed
 * (cassie_b200_last_error names the environment and the body) for a non-finite value, or a change of the world body, of a body welded to the world
 * (its geoms are static: cassie_batch_set_env_geom_pose / set_env_hfield place them per environment) or of the extra free body (its pose is qpos).
 * The rows are model inputs: reset and snapshot restore leave them alone, cassie_sim_copy copies them.  get: what every environment sees (the model's
 * offsets without rows).  clear: back to the model's offsets and the instances that ran before (constant rows the setter allocated are dropped unless
 * a model-row setter wrote them since). */
int cassie_batch_set_env_body_pos(cassie_batch_t *b, const double *pos, const unsigned char *mask);
int cassie_batch_get_env_body_pos(cassie_batch_t *b, double *pos);
int cassie_batch_clear_env_body_pos(cassie_batch_t *b);

/* Per-environment actuators (domain randomisation of actuator latency and torque saturation): for motor i of each environment
 *   ctrlrange [n][nu][2]: MuJoCo's actuator_ctrlrange (lo, hi), in both places the reference reads it -- the ctrllimited clamp of ctrl in the
 *                         actuation and motor()'s tmax, the top of the torque-speed curve and the saturation (src/cassiemujoco.c:638-664);
 *   rpm [n][nu]:          MuJoCo's actuator_user, the no-load speed in rpm (motor()'s wmax = rpm * 2 pi / 60);
 *   delay [n][nu]:        the torque delay in control ticks, 0..6: the control applied at tick k is the motor's torque of tick k - delay (6 is the
 *                         reference's TORQUE_DELAY_CYCLES, 0 applies this tick's torque).  All six slots of the delay line keep shifting whatever the
 *                         delay, so a change takes effect at once with the history in place; a variable delay is this project's extension.
 * Any of the three may be NULL (kept); mask [n] (or NULL: all) selects the environments that change.  The first call gives every environment the
 * model's values (delay 6).  0, or -1 with nothing changed (cassie_b200_last_error names the environment and the motor) for a non-finite value,
 * lo >= hi, rpm <= 0 or a delay outside 0..6.  A batch with actuator rows runs the kernel instances that read them, which also read body-offset rows:
 * without rows of its own the batch gets offset rows holding the model's values (and constant rows, as cassie_batch_set_env_body_pos does) --
 * cassie_batch_get_env_body_pos reports the model's values, cassie_batch_clear_env_body_pos puts them back instead of dropping the rows, and
 * cassie_batch_clear_env_actuators drops them unless a body-offset call has written them since.  The rows are model inputs: reset and snapshot
 * restore leave them alone, cassie_sim_copy copies them (as the rows hold them), cassie_sim_step_pd_batch honours them.  The gear, the safety layer's torque limits and the
 * encoders stay the model's.  get: what every environment sees (the model's values without rows).  clear: back to the model's actuators and the
 * kernel instances that ran before.  Device rows: cassie_batch_device_ptr(b, "actuators"), [n][ACT_W = 40] in the batch precision: lo[10], hi[10],
 * wmax[10] (rad/s), delay[10] (a real; the kernel reads it clamped to 0..6, NaN as 0, truncated) -- a write takes effect at the next launch, and the
 * rows are what the verbs work on: a masked set changes the masked environments' rows only, get reports what the rows hold (a value written on the
 * device as rpm = wmax * 60 / 2 pi and the delay as the kernel reads it). */
int cassie_batch_set_env_actuators(cassie_batch_t *b, const double *ctrlrange, const double *rpm, const int *delay, const unsigned char *mask);
int cassie_batch_get_env_actuators(cassie_batch_t *b, double *ctrlrange, double *rpm, int *delay);
int cassie_batch_clear_env_actuators(cassie_batch_t *b);
/* Per-environment mechanics (domain randomisation of the rigid-body model's inertias and the leaf springs): for each environment
 *   inertia [n][nbody][3]: MuJoCo's body_inertia, the principal moments of every body in model body order (the principal axes, body_iquat, stay the
 *                          model's);
 *   armature [n][nv]:      MuJoCo's dof_armature, the reflected rotor inertia on the diagonal of the mass matrix;
 *   stiffness [n][njnt]:   MuJoCo's jnt_stiffness, and springref [n][njnt]: its qpos_spring (the rest angle), of every hinge -- cassie.xml's shin and
 *                          heel springs.  Slide, ball and free joints keep the model's: the pelvis slides carry cassie_sim_hold's spring.
 * Any of the four may be NULL (kept); mask [n] (or NULL: all) selects the environments that change.  The first call gives every environment the model's
 * values.  0, or -1 with nothing changed (cassie_b200_last_error names the environment, the body / dof / joint and the field) for a non-finite value, a
 * negative moment, armature or stiffness, moments that break MuJoCo's rule A + B >= C for some order of the three, or a change to the world body, a body
 * welded to the world or the extra free body (its inertia and dofs), or to the stiffness or springref of a slide, ball or free joint: there the entries
 * must equal what get reports, the shared model's current values.  As in MuJoCo, the mj_setConst constants (dof_invweight0, body_invweight0, the PGS
 * scale) are not refreshed: cassie_batch_set_const computes them with each environment's inertia and armature.  A batch with mechanics rows runs the
 * kernel instances that read them, which also read actuator rows: without rows of its own the batch gets actuator rows holding the model's values (and
 * offset and constant rows through them, as cassie_batch_set_env_actuators does) -- cassie_batch_clear_env_actuators puts the model's values back
 * instead of dropping the rows, and cassie_batch_clear_env_mechanics drops them unless an actuator call has written them since.  The rows are model
 * inputs: reset and snapshot restore leave them alone, cassie_sim_copy copies them, cassie_sim_step_pd_batch honours them.  The in-kernel estimator's
 * spring model keeps the model's constants, as the robot's own estimator does.  get: what every environment sees (the model's values without rows).
 * clear: back to the model's values and the kernel instances that ran before.  Device rows: cassie_batch_device_ptr(b, "mechanics"), [n][MECH_W = 192]
 * in the batch precision: body_inertia [32][3] (model body order), then per main-tree dof armature [32], its joint's stiffness [32] and qpos_spring
 * [32], zero past nbody / nv; the kernel reads the stiffness and qpos_spring slots of hinge dofs only.  A write takes effect at the next launch, and the
 * rows are what the verbs work on: a masked set changes the masked environments' rows only, get reports what the rows hold. */
int cassie_batch_set_env_mechanics(cassie_batch_t *b, const double *inertia, const double *armature, const double *stiffness, const double *springref,
                                   const unsigned char *mask);
int cassie_batch_get_env_mechanics(cassie_batch_t *b, double *inertia, double *armature, double *stiffness, double *springref);
int cassie_batch_clear_env_mechanics(cassie_batch_t *b);
/* Per-environment contact softness (domain randomisation of how stiff and how damped the ground and the other contacts are): for each environment and
 * each geom (host model numbering, ngeom from cassie_batch_ngeom)
 *   solref [n][ngeom][2]: MuJoCo's geom_solref, standard form (timeconst, dampratio) or direct form (-stiffness, -damping);
 *   solimp [n][ngeom][5]: MuJoCo's geom_solimp (dmin, dmax, width, midpoint, power);
 *   solmix [n][ngeom]:    MuJoCo's geom_solmix, the weight of the geom's values when two geoms of equal priority mix.
 * Each contact mixes its two geoms' values as mj_contactParam does: the geom of higher priority gives its values; otherwise solimp is mixed with
 * mix = s1 / (s1 + s2) (0.5 when both solmix are below 1e-15, the other geom's values when one is), and solref too when both are in standard form, else
 * solref is the elementwise min.  condim, margin, gap and the geom priorities stay the model's; friction per geom is cassie_batch_set_geom_friction's.
 * Any of the three may be NULL (kept); mask [n] (or NULL: all) selects the environments that change.  The first call gives every environment the model's
 * values.  0, or -1 with nothing changed (cassie_b200_last_error names the environment, the geom and the field) for a non-finite value, a solref in
 * neither form (timeconst > 0 and dampratio > 0, or stiffness <= 0 and damping <= 0: mixed signs are refused), a solimp outside MuJoCo's documented
 * ranges 0 < dmin < 1, 0 < dmax < 1, width >= 0, 0 < midpoint < 1, power >= 1, or a negative solmix.  Geoms without a collision slot (visual geoms,
 * contype = conaffinity = 0) never make contact: their entries are accepted and ignored, and get reports the model's values for them (in MuJoCo,
 * writing such a geom's solref is legal and has no effect).  A batch with contact rows runs the kernel instances that read them, which also read
 * mechanics rows: without rows of its own the batch gets mechanics rows holding the model's values (and actuator, offset and constant rows through them,
 * as cassie_batch_set_env_mechanics does) -- cassie_batch_clear_env_mechanics puts the model's values back instead of dropping the rows, and
 * cassie_batch_clear_env_contact drops them unless a mechanics call has written them since.  The rows are model inputs: reset and snapshot restore
 * leave them alone, cassie_sim_copy copies them, cassie_sim_step_pd_batch honours them.  The mj_setConst constants do not depend on them.  get: what
 * every environment sees (the model's values without rows).  clear: back to the model's values and the kernel instances that ran before.  Device rows:
 * cassie_batch_device_ptr(b, "contact"), [n][CONTACT_W = 256] in the batch precision: slot k (8 values: solref [2], solimp [5], solmix) is device geom
 * k -- the collision geoms of moving bodies 0..15, then the static ones 16..31, in the order the model's candidate pairs first meet them --; slots with
 * no collision geom behind them are zero and never read.  A write takes effect at the next launch, and the rows are what the verbs work on: a masked set
 * changes the masked environments' rows only, get reports what the rows hold.  The kernel applies no clamps: a value outside the ranges above written
 * through the device pointer gives unspecified physics, but no index is derived from the row, so it cannot reach memory outside it. */
int cassie_batch_set_env_contact(cassie_batch_t *b, const double *solref, const double *solimp, const double *solmix, const unsigned char *mask);
int cassie_batch_get_env_contact(cassie_batch_t *b, double *solref, double *solimp, double *solmix);
int cassie_batch_clear_env_contact(cassie_batch_t *b);
/* Per-environment applied forces (perturbation: pushes on any body, joint-space disturbance torques), MuJoCo's mjData arrays per environment:
 * xfrc [n][nbody][6] -- xfrc_applied, force xyz and torque xyz in the world frame, applied at the body's centre of mass (xipos) -- and qfrc [n][nv] --
 * qfrc_applied, generalised forces, the extra free body's 6 dofs included.  Either may be NULL (kept); mask [n] (or NULL: all) selects the environments
 * that change.  The first call allocates the rows, zeroed.  0, or -1 with nothing changed for a non-finite value (cassie_b200_last_error names the
 * environment, the body or dof, and the field).  The world body and bodies welded to the world are accepted; their values have no effect, as in MuJoCo.
 * The values are state, as in mjData: cassie_batch_reset (masked) and cassie_sim_full_reset zero both parts, cassie_batch_clear_forces /
 * cassie_sim_clear_forces zero xfrc and keep qfrc, cassie_batch_set_const leaves both alone; snapshots (cassie_batch_get_state / set_state,
 * cassie_get_state / set_state, cassie_sim_copy) carry them -- a snapshot with rows restored into a batch without them allocates them, one without rows
 * zeroes the restored environments' rows.  The (wrench, body) slot of cassie_batch_apply_force keeps its meaning and adds to the rows: a body's total
 * xfrc_applied is its row plus the slot when the slot names it, and with rows the slot reaches the extra free body too.  The step, cassie_batch_forward
 * and cassie_sim_step_pd_batch honour the rows, and so do qacc and cacc through the solve; the dynamics rows keep MuJoCo's qfrc_bias (applied forces
 * excluded); Jacobians, the frames' contact wrenches, rays and depth images do not change.  A batch with rows runs the plain kernel instances f0404 /
 * f2404 where it would run f04 / f24, and otherwise extended instances that also read contact rows: without rows of its own the batch then gets contact
 * rows holding the model's values (and mechanics, actuator, offset and constant rows through them, as cassie_batch_set_env_contact does), dropped again
 * by enable(0) unless a contact call has written them since.  get: what the rows hold (zeros without rows); either pointer may be NULL.  enable: on = 1
 * allocates zeroed rows (for callers who only write on the device); on = 0 drops the rows and their forces, and the batch returns to the kernel
 * instances it ran before.  Device rows: cassie_batch_device_ptr(b, "applied"), [n][CASSIE_APPLIED_WIDTH] in the batch precision: xfrc_applied
 * [32][6] in model body order from CASSIE_APPLIED_XFRC, qfrc_applied [40] by dof column from CASSIE_APPLIED_QFRC (main tree 0..31, the extra free body
 * 32..37, as the DYN columns).  A write takes effect at the next launch; the kernel derives no index from the row. */
#define CASSIE_APPLIED_WIDTH 232
#define CASSIE_APPLIED_XFRC 0
#define CASSIE_APPLIED_QFRC 192
int cassie_batch_set_applied_forces(cassie_batch_t *b, const double *xfrc, const double *qfrc, const unsigned char *mask);
int cassie_batch_get_applied_forces(cassie_batch_t *b, double *xfrc, double *qfrc);
int cassie_batch_enable_applied_forces(cassie_batch_t *b, int on);
/* Per-tick traces for multi-tick launches.  A step launch of nticks control ticks normally leaves only what its last tick wrote; with a trace, every
 * tick stores k chosen columns per environment into the trace rows [n][T][k] (T = max_ticks), so that rewards and termination checks built from
 * per-tick values (foot forces, foot positions, pelvis height, motor torques, ...) can be reduced on the device after one launch.  Column c is
 * (source[c], column[c]):
 *   CASSIE_TRACE_QPOS   qpos column (0 .. nq - 1) after the tick
 *   CASSIE_TRACE_QVEL   qvel column (0 .. nv - 1) after the tick
 *   CASSIE_TRACE_OBS    observation-row column (0 .. CASSIE_OBS_WIDTH - 1) of the tick: cassie_out / state_out numbers, estimator columns included
 *   CASSIE_TRACE_AUX    derived-quantity column (0 .. CASSIE_AUX_WIDTH - 1) after the tick; needs cassie_batch_enable_aux first
 *   CASSIE_TRACE_FRAME  frame-row column (0 .. nframes * CASSIE_FRAME_WIDTH - 1) after the tick; needs cassie_batch_set_frames first
 * Slot s holds what the rows would hold had the launch stopped after that tick (what cassie_batch_get_* returns after a 1-tick launch).  A launch of
 * nticks <= T writes slots 0 .. nticks - 1 and leaves the others alone; a longer one keeps its last T ticks, in order.  cassie_sim_step_pd_batch
 * writes slot 0.  The rows are an output: only step launches write them; forward, query, set_const, Jacobian and dynamics launches, resets, set_state,
 * reset_where and snapshots leave them alone.  set_trace allocates the rows (zeroed), so that a step allocates and synchronises nothing; k = 0 drops
 * the trace.  0, or -1 with nothing changed (cassie_b200_last_error says why) for: an unknown source, a column outside its source's range, k outside
 * 0 .. CASSIE_TRACE_MAX, max_ticks < 1 with k > 0, an aux or frame column without those rows, the batch of a cassie_sim_t.  While a traced column
 * reads them, cassie_batch_enable_aux(b, 0) and cassie_batch_set_frames are refused.
 * A traced batch runs the F_TC twins of the extended applied-force instances: it carries applied-force rows (zeroed ones when it has none, dropped
 * again by k = 0 unless an applied-force verb has written them since) and, through them, model-valued contact rows as with applied forces; the
 * physics is bitwise that of the same batch without a trace.  trace_ticks: the slots the last step launch wrote (min(nticks, T); 0 before the first).
 * get_trace: synchronous host copy [n][T][k] doubles.  Device rows: cassie_batch_device_ptr(b, "trace"), [n][T * k] in the batch precision
 * (cassie_batch_row_width(b, "trace") = T * k). */
#define CASSIE_TRACE_QPOS 0
#define CASSIE_TRACE_QVEL 1
#define CASSIE_TRACE_OBS 2
#define CASSIE_TRACE_AUX 3
#define CASSIE_TRACE_FRAME 4
#define CASSIE_TRACE_MAX 64
int cassie_batch_set_trace(cassie_batch_t *b, const int *source, const int *column, int k, int max_ticks);
int cassie_batch_trace_ticks(const cassie_batch_t *b);
int cassie_batch_get_trace(cassie_batch_t *b, double *out);
/* Contact lists for the batch: every environment's MuJoCo contact list (d->contact) and mj_contactForce, as the reference's users read them through
 * cassie_sim_mjdata and its own queries are built on them (src/cassiemujoco.c:1586-1606, 1781-1898): which geom a foot touched and where, the normal
 * on a slope, the penetration depth, the friction the solver used, the contact points and frames a contact-aware controller needs.  With contact rows
 * enabled, every step launch (cassie_sim_step_pd_batch's chunk launches included) and every forward launch (forward_where too: the selected environments
 * only) fills one row per environment with the contacts of the launch's last sub-step -- the state that sub-step started from, which is what the
 * reference's queries read after a step -- that entered the solve, in MuJoCo's order, within the capacities of 12 contacts and 48 constraint rows.
 * Query, set_const, Jacobian, dynamics and inverse launches, resets, set_state, reset_where and snapshots leave the rows alone (they are an output;
 * a restore followed by forward_where refreshes them).  Row [CASSIE_CON_WIDTH] in the batch precision: CASSIE_CON_HEAD header reals -- [0] contacts
 * listed, [1] contacts the collision stage found, [2] contacts dropped at the capacities (found - listed; the increment of counters[4]), the rest zero --
 * then CASSIE_CON_MAX slots of CASSIE_CON_SLOT reals, slot k at CASSIE_CON_HEAD + CASSIE_CON_SLOT * k:
 *   CASSIE_CON_GEOM1, GEOM2  geom ids in the model's numbering (cassie_batch_id2name(b, "geom", id)); -1 in unused slots
 *   CASSIE_CON_DIM           condim
 *   CASSIE_CON_DIST          contact.dist (negative: penetration)
 *   CASSIE_CON_POS   [3]     contact.pos, world frame
 *   CASSIE_CON_FRAME [9]     contact.frame, row-major: row 0 the normal, from geom1 to geom2; rows 1 and 2 the tangents
 *   CASSIE_CON_FORCE [6]     mj_contactForce in the contact frame: normal, two tangential, three torques (zero at condim <= 3).  The force geom2 feels
 *                            in the world frame is frame' force[0..2]; geom1 feels its negative
 *   CASSIE_CON_MU            the friction the pyramid used: the pair's mixed friction, from the per-environment friction rows where the batch has them
 *   CASSIE_CON_EFC           contact.efc_address: the contact's first constraint row (the equality and limit rows come first)
 * Unused slots are zero apart from the geom ids.  enable_contacts(b, 1) allocates zeroed rows, so that a launch allocates and synchronises nothing;
 * enable_contacts(b, 0) frees them.  A batch with contact rows runs the F_CL twins of the extended applied-force instances: it carries applied-force
 * and contact rows (model-valued ones when it has none, dropped again by enable_contacts(b, 0) unless a verb has written them since), and its physics
 * is bitwise that of the same batch without contact rows.  A batch with a per-tick trace refuses contact rows and a batch with contact rows refuses a
 * trace.  get_contacts: synchronous host copy [n][CASSIE_CON_WIDTH] doubles.  Device rows: cassie_batch_device_ptr(b, "contacts"),
 * cassie_batch_row_width(b, "contacts") = CASSIE_CON_WIDTH.  0, or -1 (cassie_b200_last_error says why). */
#define CASSIE_CON_HEAD 8
#define CASSIE_CON_SLOT 24
#define CASSIE_CON_MAX 12
#define CASSIE_CON_WIDTH 296
#define CASSIE_CON_GEOM1 0
#define CASSIE_CON_GEOM2 1
#define CASSIE_CON_DIM 2
#define CASSIE_CON_DIST 3
#define CASSIE_CON_POS 4
#define CASSIE_CON_FRAME 7
#define CASSIE_CON_FORCE 16
#define CASSIE_CON_MU 22
#define CASSIE_CON_EFC 23
int cassie_batch_enable_contacts(cassie_batch_t *b, int on);
int cassie_batch_get_contacts(cassie_batch_t *b, double *out);
/* Sensor models, drawn in the step kernel: what the controller, the safety layer, the encoder filters and the estimator of every step tick measure.
 * Each tick the controller stage takes last step's sensordata and measures:
 *   encoder c (cassie_out order: 10 drives, then 6 joints)   true + offset[c] + n_c (output radians; a drive's motor-side value moves by gear times
 *                                                            that), then the encoder's quantisation and filters as before
 *   IMU orientation                                          q (x) q_m (x) normalise(1, (n_16, n_17, n_18) / 2)
 *   gyro / accelerometer                                     R_m' v + bias + (n_19..21) / (n_22..24), clamped at the model's sensor cutoffs
 *   magnetometer                                             R_m' m
 * where q_m is the environment's IMU mount quaternion.  MuJoCo's sensordata (rows, aux, frames, rays, cameras) keeps the true values.  Noise: channel c
 * takes 64-bit word c % 4 of the Philox-4x64-10 block with key (seed, 0) and counter (t, c / 4, 0, 0), t = the environment's counter + the tick of the
 * launch; n = std * C * (u0 + u1 + u2 + u3 - 131070) over the word's four 16-bit parts, C = 1 / sqrt((65536^2 - 1) / 3): zero mean, unit variance
 * times std, kurtosis 2.7, tails cut at 3.46 std (Irwin-Hall with four terms; integer operations and correctly rounded multiplies, so every build
 * draws the same bits).  Step launches advance the counter by their tick count; other launches, resets, reset_where and snapshots leave it alone, so
 * a new episode never replays old noise.  To replay a stretch, save and restore the counter (device rows "sensor_rng").
 * set_env_sensors: enc_offset [n][16], enc_noise [n][16] (std), imu_quat [n][4] (w x y z, normalised on write), imu_bias [n][6] (gyro, accelerometer),
 * imu_noise [n][9] (std of orientation in rad, gyro, accelerometer); NULL keeps a part, only masked environments change.  The first call allocates
 * the zero model (zeros, identity mount; bitwise the batch without rows) and generator rows as seed_sensors(b, 0, NULL) seeds them.  A non-finite
 * value, a negative std or a zero quaternion is refused with nothing changed, and the error names the environment, channel and field.  The rows are a
 * model input: resets and snapshot restores leave them alone, cassie_sim_copy copies them and the generator rows, cassie_sim_step_pd_batch honours
 * them.  A batch with rows runs the F_SN twins of the applied-force instances (carrying zero applied-force rows when it has none) and refuses a
 * per-tick trace or contact lists, as they refuse it.  get: NULL parts are skipped; the zero model without rows.  clear: drops the rows, back to the
 * instances that ran before.  seed_sensors: environment i gets key seed + i and counter 0 (masked environments only).  get_sensor_rng: key and
 * counter [n] each.  Device rows: cassie_batch_device_ptr(b, "sensors") [n][CASSIE_SENSOR_WIDTH] in the batch precision, laid out as CASSIE_SN_*, and
 * "sensor_rng" [n][4] int32 (key lo, hi, counter lo, hi); a write takes effect at the next launch.  0, or -1 (cassie_b200_last_error says why). */
#define CASSIE_SENSOR_WIDTH 52
#define CASSIE_SN_ENC_OFF 0
#define CASSIE_SN_ENC_STD 16
#define CASSIE_SN_QUAT 32
#define CASSIE_SN_ORI_STD 36
#define CASSIE_SN_GYRO_BIAS 39
#define CASSIE_SN_GYRO_STD 42
#define CASSIE_SN_ACC_BIAS 45
#define CASSIE_SN_ACC_STD 48
int cassie_batch_set_env_sensors(cassie_batch_t *b, const double *enc_offset, const double *enc_noise, const double *imu_quat, const double *imu_bias,
                                 const double *imu_noise, const unsigned char *mask);
int cassie_batch_get_env_sensors(cassie_batch_t *b, double *enc_offset, double *enc_noise, double *imu_quat, double *imu_bias, double *imu_noise);
int cassie_batch_clear_env_sensors(cassie_batch_t *b);
int cassie_batch_seed_sensors(cassie_batch_t *b, unsigned long long seed, const unsigned char *mask);
int cassie_batch_get_sensor_rng(cassie_batch_t *b, unsigned long long *seed, unsigned long long *counter);
/* Names of the compiled model's objects, as mj_name2id / mj_id2name give them (the reference's cassie_sim_mj_name2id, src/cassiemujoco.c:2194-2246):
 * type "body" (or "xbody"), "joint", "geom", "site" or "camera".  name2id: the id, or -1 for an unknown or empty name; id2name: the name, or NULL for
 * an id out of range or an unnamed object (the string lives as long as the batch).  Both return -1 / NULL with a recorded error for mj_name2id's other
 * kinds (actuators, equalities, meshes, ...: the compiled model keeps no names of them) and for an unknown type.  cassie_sim_mj_name2id is the same
 * lookup on a cassie_sim_t. */
int cassie_batch_name2id(const cassie_batch_t *b, const char *type, const char *name);
const char *cassie_batch_id2name(const cassie_batch_t *b, const char *type, int id);
/* The controller-stage state of every environment, as the reference's cassie_sim_t holds it: the torque delay line torque_delay [n][10][6] (slot 0
 * newest), the drive encoders' integer FIR taps drive_filter [n][10][9], the joint encoders' IIR filters joint_x [n][6][4] and joint_y [n][6][3].
 * NULL parts are skipped; set changes masked environments only (mask NULL: all).  They are state: reset, snapshots and cassie_sim_copy carry them. */
int cassie_batch_get_actuator_state(cassie_batch_t *b, double *torque_delay, int *drive_filter, double *joint_x, double *joint_y);
int cassie_batch_set_actuator_state(cassie_batch_t *b, const double *torque_delay, const int *drive_filter, const double *joint_x, const double *joint_y,
                                    const unsigned char *mask);

/* zero-copy access for a PyTorch / DLPack caller: device pointer of a state array ("qpos" [n][36], "qvel" [n][32],
 * "pd" [n][52], "obs" [n][112], "xfrc" [n][8], "aux" [n][64], "frames" [n][count * 20], "acc" [n][40 + 8 count], "actuators" [n][40], "mechanics" [n][192], "contact" [n][256], "applied" [n][232], "trace" [n][T * k], "contacts" [n][296], "inv_qacc" [n][32] ([n][40]), "inv" [n][96]; the inverse rows are allocated by the request) in the batch precision, "terrain" [n] int32; the stream all work is enqueued on
 * (cudaStream_t). */
void *cassie_batch_device_ptr(cassie_batch_t *b, const char *field);
void cassie_batch_set_stream(cassie_batch_t *b, void *cuda_stream);
void *cassie_batch_get_stream(cassie_batch_t *b);
int cassie_batch_precision(const cassie_batch_t *b);
/* row width (in elements) of a device array named as in cassie_batch_device_ptr: qpos 36 (44 with the extra free body of cassie_tray_box.xml), qvel 32 (40) */
int cassie_batch_row_width(const cassie_batch_t *b, const char *field);
/* per-env solver statistics of the last sub-step: int [n][8] = nefc, ncon, nlimit, PGS iterations, dropped contacts, 0,0,0 */
void cassie_batch_get_counters(cassie_batch_t *b, int *out);
/* launches issued since init (bench.py's gpu_launches) */
long cassie_batch_launch_count(const cassie_batch_t *b);
/* test hook: stage-by-stage intermediates of env `env` from the last sub-step (DevModel debug layout, doubles) */
int cassie_batch_debug_dump(cassie_batch_t *b, int env, double *out, int n);
/* last error message of this thread ("" if none) */
const char *cassie_b200_last_error(void);

#ifdef __cplusplus
}
#endif
#endif /* CASSIE_B200_H */
