// step_kernel.cuh -- the fused step kernel (one warp per environment) and its argument block.  Included by step_inst.cu, which is compiled once per
// kernel instance (precision x plain / extended x model features) so that the instances build in parallel and each carries only the code its
// models need, and by cassie_b200.cu for the argument types; the instances are reached through cassie_step_entry_<tag>() function pointers.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include "devmodel.h"
#include "estimator_host.h"
#include "step_core.inl"

namespace cassie {

#ifdef CASSIE_DBG_ALL
constexpr bool DBG_IN_ALL_INSTANCES = true;
#else
constexpr bool DBG_IN_ALL_INSTANCES = false;
#endif

template <typename real> struct EnvArrays {
  real *qpos, *qvel, *qacc_ws, *cst, *pd, *xfrc, *obs, *dbg, *qM, *aux, *cenv, *task, *gait; const real *pd_host; real *obs_host; double *est; int *dfilt, *counters, *ticket; const float *hfield; const unsigned char *mask; int cta_sync, nsub, warp_stride, env0; int n, n_terrain, qpos_w, qvel_w, ystride, xb; size_t hfield_stride;
  const real *genv;   // [n][GEOM_ENV_W] per-environment static-geom placement or null (read by the F_EG instances only); last, so the other members keep their offsets
  const real *ftab; real *frames; int nfr;   // frame table [nfr][FT_W] and rows [n][nfr][FRAME_W] (read by the F_FR instances only); after genv for the same reason
  real *jac; int jfr;                         // mode 4: Jacobian rows [n][FRAME_JAC_W] of frame jfr (F_FR instances)
  real *dyn;                                  // mode 5: dynamics rows [n][DYN_W] (F_FR instances)
  real *acc;                                  // modes 0 / 1: acceleration rows [n][acc_width(nfr)] or null (F_FR instances)
  const int *terrain;                         // [n] bank entry of each environment, read mod n_terrain (F_TR instances)
  const real *bpos;                           // [n][BP_W] body offsets of each environment (F_BP instances)
  const real *act;                            // [n][ACT_W] actuators of each environment (F_AC instances)
  const real *mech;                           // [n][MECH_W] inertia, armature and hinge springs of each environment (F_MC instances)
  const real *contact;                        // [n][CONTACT_W] solref, solimp and solmix per collision geom of each environment (F_CT instances)
  const real *applied;                        // [n][APPLIED_W] xfrc_applied and qfrc_applied of each environment (F_XF instances)
  TraceArgs<real> trace;                      // [n][T][k] per-tick trace rows and their column table (F_TC instances)
  real *inv;                                  // mode 6: inverse rows [n][INV_W] (F_FR instances); the launch's qacc_ws is the batch's inverse input, its
                                              // dbg, cst and counters are scratch rows
  ContactListArgs<real> cl;                   // [n][CON_W] contact-list rows and the device-to-model geom ids [MGT] (F_CL instances); last, so that
                                              // the model block (DevModel, which with 16 warps fills the shared memory) does not grow
  SensorArgs<real> sn;                        // [n][SN_W] sensor-model rows and [n][SR_W] generator rows (F_SN instances)
};

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

// stage `bytes` (multiple of 16) from global to shared with one TMA bulk copy; all threads of the CTA return after it landed
__device__ __forceinline__ void tma_stage(void *dst_smem, const void *src_gmem, uint32_t bytes, uint64_t *bar) {
  const uint32_t bar_a = smem_u32(bar), dst_a = smem_u32(dst_smem);
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar_a), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bytes) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_a), "l"(src_gmem), "r"(bytes), "r"(bar_a) : "memory");
  }
  asm volatile(
      "{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(bar_a), "r"(0) : "memory");
}

template <typename real> __host__ __device__ constexpr size_t model_bytes() { return (sizeof(DevModel<real>) + 127) / 128 * 128; }
template <typename real> __host__ __device__ constexpr size_t warp_bytes(int ystride, bool ext) { return ((size_t)(ext ? scratch_reals_ext(ystride) : scratch_reals(ystride)) * sizeof(real) + 127) / 128 * 128; }

// mode 0: step nticks; mode 1: mj_forward only; 2 / 3 / 4 / 5 / 6: query, set_const, frame Jacobian, dynamics row, inverse row (see mj_substep).  INST: 0 plain instance, 1 extended instance (per-env constants, derived quantities, task PD, set_const,
// estimator), 2 plain instance + estimator stage (what cassie_sim_step_pd_batch runs when nothing else asks for the extended one)
template <typename real, int INST, int FEAT>
__global__ void __launch_bounds__(512) cassie_step_kernel(const DevModel<real> *__restrict__ gmodel, EnvArrays<real> A, int nticks, int mode) {
  extern __shared__ __align__(128) unsigned char smem_raw[];
  __shared__ __align__(8) uint64_t bar;
  DevModel<real> *cmp = reinterpret_cast<DevModel<real> *>(smem_raw);
  tma_stage(cmp, gmodel, (uint32_t)model_bytes<real>(), &bar);
  const int warp = threadIdx.x >> 5, l = threadIdx.x & 31;
  real *sm = reinterpret_cast<real *>(smem_raw + model_bytes<real>() + warp * A.warp_stride);   // warp_stride = warp_bytes(ystride, instance), precomputed on the host: cheap to rematerialise under register pressure
  const int qw = (FEAT & F_XB) ? A.qpos_w : QPOS_W_MAIN, vw = (FEAT & F_XB) ? A.qvel_w : QVEL_W_MAIN;
  const DevModel<real> &cm = *cmp;
  // persistent CTAs with a static round-robin schedule: in round r CTA b owns environments [(r gridDim + b) nwarps, ... + nwarps), one per warp.  The
  // grid is sized to the resident CTAs, the environments cost about the same, and a static schedule lets every warp pull the rows of its NEXT
  // environment towards L2 while it steps the current one.  (Multi-tick launches: the CTA's warps walk the stages together, STAGE_SYNC, so that
  // they share instruction-cache lines -- the kernel is ~200 KB of code, several times the L1.5.)
  const int nwarps = blockDim.x >> 5, sync_on = (mode == 0 && (nticks > 1 || (A.cta_sync & 32))) ? (A.cta_sync & 31) : 0;   // bit 5: also in single-tick launches
  const int stride = gridDim.x * nwarps;
  for (int base = blockIdx.x * nwarps; base < A.n; base += stride) {
    const int env = A.env0 + base + warp;   // a launch covers environments [env0, env0 + n)
    if (!(A.cta_sync & 64)) __syncthreads();   // the warps of a CTA start every round together: they then share instruction-cache lines through the round (measured: 16 384
                       // environments, 7 rounds, -20 % without it), and the multi-tick rendezvous counts below assume it
    { const int nenv = base + warp + stride < A.n ? env + stride : 0x7fffffff;   // warm L2 with the next round's state rows of this warp (about 2 KB per environment, one 128-byte line per lane)
      if (nenv != 0x7fffffff && mode == 0) {
        const char *p = nullptr;
        if (l < 6) p = (const char *)(A.cst + (size_t)nenv * CST_W) + 128 * l * (sizeof(real) / 4);
        else if (l < 9) p = (const char *)(A.dfilt + (size_t)nenv * DFILT_W) + 128 * (l - 6);
        else if (l < 11) p = (const char *)(A.pd + (size_t)nenv * PD_W) + 128 * (l - 9) * (sizeof(real) / 4);
        else if (l < 13) p = (const char *)(A.qpos + (size_t)nenv * qw) + 128 * (l - 11) * (sizeof(real) / 4);
        else if (l < 15) p = (const char *)(A.qvel + (size_t)nenv * vw) + 128 * (l - 13) * (sizeof(real) / 4);
        else if (l < 17) p = (const char *)(A.qacc_ws + (size_t)nenv * vw) + 128 * (l - 15) * (sizeof(real) / 4);
        else if (l == 17) p = (const char *)(A.xfrc + (size_t)nenv * XFRC_W);
        if (p) asm volatile("prefetch.global.L2 [%0];" ::"l"(p));
      } }
    const bool active = base + warp < A.n && !(A.mask && !A.mask[env]);   // masked launches (reset / set_const of a subset)
    if (!active) {   // keep the rendezvous count of the working warps
      if (sync_on) { const int per = __popc(sync_on); for (int i = 0; i < nticks * (A.nsub > 0 ? A.nsub : cm.nsub) * per; ++i) __syncthreads(); }
      continue;
    }
    // warm the L2/L1 path of the rows that are addressed in place later (controller state, PD row, FIR taps)
    if (l < 6) asm volatile("prefetch.global.L2 [%0];" ::"l"(A.cst + (size_t)env * CST_W + 32 * l));
    else if (l < 9) asm volatile("prefetch.global.L2 [%0];" ::"l"(A.dfilt + (size_t)env * DFILT_W + 32 * (l - 6)));
    else if (l < 11) asm volatile("prefetch.global.L2 [%0];" ::"l"(A.pd + (size_t)env * PD_W + 32 * (l - 9)));
    else if (l == 11) asm volatile("prefetch.global.L2 [%0];" ::"l"(A.xfrc + (size_t)env * XFRC_W));
    // optional zero-copy input: this environment's motor-PD row straight from mapped host memory into its device row (the AoS entry point
    // uses one DMA instead: 2 x 4096 small PCIe reads at kernel start were measured slower than the copy engine; kept for C2C-attached hosts)
    if (A.pd_host) { for (int i = l; i < PD_W; i += 32) A.pd[(size_t)env * PD_W + i] = A.pd_host[(size_t)env * PD_W + i]; }
    // state rows: qpos to shared memory, qvel / warm start one value per lane; everything else is addressed in place
    for (int i = l; i < qw; i += 32) sm[S_QPOS + i] = (mode == 3) ? cm.qpos0[i] : A.qpos[(size_t)env * qw + i];   // set_const works at the reference configuration
    real qvel = A.qvel[(size_t)env * vw + l], qacc_ws = A.qacc_ws[(size_t)env * vw + l], xqvel = 0, xqacc_ws = 0;
    if ((FEAT & F_XB) && A.xb >= 0 && l < 6) { xqvel = A.qvel[(size_t)env * vw + 32 + l]; xqacc_ws = A.qacc_ws[(size_t)env * vw + 32 + l]; }
    __syncwarp();
    EnvPtrs<real> E;   // (E.dbg: the stage dumps are compiled into the extended instance only; batches created with debug = 1 run that one)
    E.cst = A.cst + (size_t)env * CST_W; E.dfilt = A.dfilt + (size_t)env * DFILT_W; E.pd = A.pd + (size_t)env * PD_W; E.xfrc = A.xfrc + (size_t)env * XFRC_W; E.task = A.task ? A.task + (size_t)env * TASK_W : nullptr; E.gait = A.gait ? A.gait + (size_t)env * GAIT_W : nullptr;
    E.hfield = A.hfield ? A.hfield + (size_t)(env % A.n_terrain) * A.hfield_stride : nullptr;
    if constexpr ((FEAT & F_TR) != 0) { if (A.hfield) E.hfield = A.hfield + (size_t)((unsigned)A.terrain[env] % (unsigned)A.n_terrain) * A.hfield_stride; }   // any value in the row stays inside the bank
    E.obs = A.obs + (size_t)env * OBS_W; E.qM = A.qM + (size_t)env * 2 * NM_MAX; E.dbg = (DBG_IN_ALL_INSTANCES || INST == 1) && A.dbg ? A.dbg + (size_t)env * D_SIZE : nullptr; E.counters = A.counters + (size_t)env * 8;
    E.aux = A.aux ? A.aux + (size_t)env * AUX_W : nullptr; E.cenv = A.cenv ? A.cenv + (size_t)env * CE_W : nullptr; E.cta_sync = sync_on; E.nsub = A.nsub;
    E.est = A.est ? A.est + (size_t)env * EST_W : nullptr; E.est_out = E.obs + OB_EST_OUT;
    if (FEAT & F_EG) { E.genv = A.genv; E.env = env; }   // the row address is formed where the collision stage reads it: no pointer held across the step
    if (FEAT & F_FR) { E.ftab = A.ftab; E.frames = A.frames; E.nfr = A.nfr; E.jac = A.jac; E.jfr = A.jfr; E.env = env; }   // likewise the frame rows, at each frame stage
    if (FEAT & F_BP) E.env = env;   // the body-offset rows likewise, at the kinematics, from the kernel parameter A.bpos
    if (FEAT & F_AC) E.env = env;   // and the actuator rows, at the motor stage and the actuation, from A.act
    if (FEAT & F_MC) E.env = env;   // and the mechanics rows, at the cinert, CRB and passive phases, from A.mech
    if (FEAT & F_CT) E.env = env;   // and the contact rows, at the contact rows' constants, from A.contact
    if (FEAT & F_XF) E.env = env;   // and the applied-force rows, at the bias sum, the applied dof forces and the extra body's acceleration, from A.applied
    if (FEAT & F_TC) E.env = env;   // and the trace rows, after every tick, from A.trace
    if (FEAT & F_CL) E.env = env;   // and the contact-list rows, in the last sub-step, from A.cl
    if (FEAT & F_SN) E.env = env;   // and the sensor-model and generator rows, at the controller stage, from A.sn
    step_env<real, INST == 1, FEAT, INST >= 1>(cm, sm, E, qvel, qacc_ws, xqvel, xqacc_ws, nticks, mode, (FEAT & F_BP) ? A.bpos : (const real *)0, (FEAT & F_AC) ? A.act : (const real *)0,
                                               (FEAT & F_MC) ? A.mech : (const real *)0, (FEAT & F_CT) ? A.contact : (const real *)0, (FEAT & F_XF) ? A.applied : (const real *)0,
                                               (FEAT & F_TC) ? A.trace : TraceArgs<real>{}, (FEAT & F_CL) ? A.cl : ContactListArgs<real>{},
                                               (FEAT & F_SN) ? A.sn : SensorArgs<real>{});
    __syncwarp();
    if (mode >= 2) {   // query / set_const / frame Jacobian / dynamics / inverse: only the aux row / the constant row / the Jacobian row / the dynamics row / the inverse row is written
      if constexpr ((FEAT & F_FR) != 0) {   // from what mode 5's / mode 6's sub-step left in shared memory (mode 6: and in its scratch rows)
        if (mode == 5) dynamics_row(cm, sm, A.dyn, A.cenv, env, (FEAT & F_XB) ? cm.xb : -1);
        else if (mode == 6) inverse_row(cm, sm, A.inv, A.cenv, A.dbg, A.qacc_ws, A.counters, env);
      }
      continue;
    }
    for (int i = l; i < qw; i += 32) A.qpos[(size_t)env * qw + i] = sm[S_QPOS + i];
    A.qvel[(size_t)env * vw + l] = qvel; A.qacc_ws[(size_t)env * vw + l] = qacc_ws;
    if ((FEAT & F_XB) && A.xb >= 0 && l < 6) { A.qvel[(size_t)env * vw + 32 + l] = xqvel; A.qacc_ws[(size_t)env * vw + 32 + l] = xqacc_ws; }
    // ... and its observation row goes back the same way as soon as the environment is done, overlapped with the environments still stepping (sending it
    // right after the controller stage, before the physics, was measured: no end-to-end gain, -2.8 % on every instance from the longer-lived pointer)
    if (A.obs_host) { for (int i = l; i < OBS_W; i += 32) A.obs_host[(size_t)env * OBS_W + i] = A.obs[(size_t)env * OBS_W + i]; }
    if constexpr ((FEAT & F_FR) != 0) { if (A.acc) accel_row(cm, sm, A.acc, A.ftab, A.frames, A.nfr, env, (FEAT & F_XB) ? cm.xb : -1); }   // from what the last sub-step left in shared memory
    __syncwarp();
  }
}

}  // namespace cassie
