// cassie_b200.cu -- CUDA kernels (sm_90a) and the C-ABI of the batched Cassie stepper.  See include/cassie_b200.h.
//
// Kernel shape: one warp per environment; a CTA of WPB warps first stages the model constant block into shared memory with
// a TMA bulk copy (cp.async.bulk + mbarrier, SASS: UBLKCP), then every warp loads its environment's state rows from HBM
// (coalesced, one row per array), advances `nticks` control ticks entirely on chip (step_core.inl) and writes the rows back.
#include <cuda_runtime.h>
#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>
#include <omp.h>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/cassie_b200.h"
#include "devbuild.h"
#include "estimator_host.h"
#include "step_kernel.cuh"
#include "step_select.h"
#include "env_rows.h"
#include "raycast.inl"
#include "camera_set.inl"
#include "reset.inl"
#include "loops.inl"
#include "ik.inl"

// the step-kernel instances live in their own translation units (step_inst.cu, one compilation per line of step_instances.inc)
#define STEP_INSTANCE(tag) extern "C" const void *cassie_step_entry_##tag(void);
#include "step_instances.inc"
#undef STEP_INSTANCE

namespace cassie {

template <typename real> cudaError_t launch_raycast(const RayArgs<real> &A, int device, cudaStream_t stream);   // raycast.cu
template <typename real> cudaError_t launch_camera(const CamArgs<real> &A, int device, cudaStream_t stream);   // camera.cu
template <typename real> cudaError_t launch_camera_set(const CamSetArgs<real> &A, int device, cudaStream_t stream);   // camera_set.cu
template <typename real> cudaError_t launch_reset(const ResetArgs &A, int device, cudaStream_t stream);       // reset.cu
template <typename real> cudaError_t launch_loops(const LoopArgs<real> &A, int device, cudaStream_t stream);   // loops.cu
template <typename real> cudaError_t launch_ik(const IkArgs<real> &A, int device, cudaStream_t stream);         // ik.cu

static constexpr StepInstance STEP_INSTANCES[] = {
#define STEP_INSTANCE(tag) step_instance(#tag, cassie_step_entry_##tag),
#include "step_instances.inc"
#undef STEP_INSTANCE
};

template <typename real> static StepChoice select_step(int kind, int feat) {
  return step_select(STEP_INSTANCES, (int)(sizeof STEP_INSTANCES / sizeof STEP_INSTANCES[0]), std::is_same<real, double>::value, kind, feat);
}

// cassie_sim_centroid_inertia (src/cassiemujoco.c:1647-1687) from one dynamics row: m = M[0][0], I_p = M[3:6, 3:6], r = the row's centre-of-mass offset
// (DY_RCM).  The diagonal is I_p - m (r_j^2 + r_k^2); the off-diagonals are I_p[i][j] - m r_i r_j, with the reference's sign (the parallel-axis
// theorem has + there), taken from the lower triangle as the reference does.
template <typename real> static void centroid_inertia(const real *row, double Icm[9]) {
  double Ip[3][3], r[3]; const double m = (double)row[DY_M];
  for (int i = 0; i < 3; i++) { r[i] = (double)row[DY_RCM + i]; for (int j = 0; j < 3; j++) Ip[i][j] = (double)row[DY_M + (i + 3) * DY_COLS + j + 3]; }
  double Ic[3][3];
  Ic[0][0] = Ip[0][0] - m * (r[1] * r[1] + r[2] * r[2]);
  Ic[1][1] = Ip[1][1] - m * (r[2] * r[2] + r[0] * r[0]);
  Ic[2][2] = Ip[2][2] - m * (r[0] * r[0] + r[1] * r[1]);
  Ic[0][1] = Ic[1][0] = Ip[1][0] - m * r[1] * r[0];
  Ic[1][2] = Ic[2][1] = Ip[2][1] - m * r[2] * r[1];
  Ic[2][0] = Ic[0][2] = Ip[2][0] - m * r[2] * r[0];
  for (int i = 0; i < 3; i++) for (int j = 0; j < 3; j++) Icm[3 * i + j] = Ic[i][j];
}

static thread_local std::string g_err;
static void set_err(const std::string &e) { g_err = e; fprintf(stderr, "cassie_b200: %s\n", e.c_str()); }
#define CUDA_OK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { set_err(std::string(#call) + ": " + cudaGetErrorString(e_)); return false; } } while (0)

// CPUs this process may actually use: the affinity mask clipped by the cgroup CPU quota (a container on a 128-thread host may own 16)
static int effective_cpus() {
  int hw = omp_get_num_procs();
  long quota = -1, period = 0;
  if (FILE *f = fopen("/sys/fs/cgroup/cpu.max", "r")) { char q[64]; if (fscanf(f, "%63s %ld", q, &period) == 2 && strcmp(q, "max")) quota = atol(q); fclose(f); }
  else {
    if (FILE *g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_quota_us", "r")) { if (fscanf(g, "%ld", &quota) != 1) quota = -1; fclose(g); }
    if (FILE *g = fopen("/sys/fs/cgroup/cpu/cpu.cfs_period_us", "r")) { if (fscanf(g, "%ld", &period) != 1) period = 0; fclose(g); }
  }
  if (quota > 0 && period > 0) { const int c = (int)((quota + period - 1) / period); if (c >= 1 && c < hw) hw = c; }
  return hw < 1 ? 1 : hw;
}
// host pack / unpack threads of the AoS entry point.  The OpenMP workers busy-wait between the call's parallel regions, so the team burns its CPUs for the
// whole call: by default two of the CPUs the process may use (affinity mask clipped by the cgroup quota) are left to the CUDA driver's and the caller's
// own threads -- a team as large as the quota gets the whole cgroup throttled
static int aos_thread_count() {
  const char *e = getenv("CASSIE_B200_AOS_THREADS"); const int hw = effective_cpus();
  int t = e ? atoi(e) : (hw > 4 ? hw - 2 : hw); if (t > 32) t = 32; if (t > hw) t = hw; return t < 1 ? 1 : t;
}

// cassie_integrate_pos for the whole batch (mj_integratePos, src/cassiemujoco.c:1183-1189): the HBM-bound kernel.
// A tile of ITILE consecutive environments is one contiguous chunk of the qpos array and one of the qvel array.  Persistent CTAs
// stream tiles through an ISTAGES-deep shared-memory ring: TMA bulk loads (cp.async.bulk -> mbarrier), in-place arithmetic,
// TMA bulk store of the qpos chunk.  Algorithmic traffic per env: read qpos + qvel, write qpos = (36 + 32 + 36) reals.
constexpr int ITILE = 64, ISTAGES = 4;
template <typename real> __host__ __device__ constexpr size_t itile_bytes(int qw, int vw) { return (size_t)ITILE * (qw + vw) * sizeof(real); }
template <typename real>
__global__ void __launch_bounds__(256) cassie_integrate_kernel(const DevModel<real> *__restrict__ gmodel, real *__restrict__ qpos, const real *__restrict__ qvel, int n, int QPOS_W, int QVEL_W) {
  extern __shared__ __align__(128) unsigned char ibuf[];
  __shared__ __align__(8) uint64_t bar[ISTAGES];
  __shared__ int ns, nb, sq_adr[MJ + 4], sd_adr[MJ + 4], bq_adr[MJ], bd_adr[MJ];
  __shared__ real h;
  const int ntiles = (n + ITILE - 1) / ITILE;
  if (threadIdx.x == 0) {
    int a = 0, b = 0;
    for (int j = 0; j < gmodel->njnt; ++j) {
      const int t = gmodel->jnt_type[j];
      if (t >= 2) { sq_adr[a] = gmodel->jnt_qposadr[j]; sd_adr[a] = gmodel->jnt_dofadr[j]; ++a; } else if (t == 1) { bq_adr[b] = gmodel->jnt_qposadr[j]; bd_adr[b] = gmodel->jnt_dofadr[j]; ++b; }
      else {   // free joint: three translations like slides, the quaternion like a ball joint
        for (int k = 0; k < 3; ++k) { sq_adr[a] = gmodel->jnt_qposadr[j] + k; sd_adr[a] = gmodel->jnt_dofadr[j] + k; ++a; }
        bq_adr[b] = gmodel->jnt_qposadr[j] + 3; bd_adr[b] = gmodel->jnt_dofadr[j] + 3; ++b;
      }
    }
    ns = a; nb = b; h = gmodel->timestep;
    for (int s = 0; s < ISTAGES; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(&bar[s])), "r"(1));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  auto issue_load = [&](int stage, int tile) {   // thread 0 only
    const int cnt = min(ITILE, n - tile * ITILE);
    const uint32_t bq = (uint32_t)(cnt * QPOS_W * sizeof(real)), bv = (uint32_t)(cnt * QVEL_W * sizeof(real));
    unsigned char *dst = ibuf + (size_t)stage * itile_bytes<real>(QPOS_W, QVEL_W);
    const uint32_t bar_a = smem_u32(&bar[stage]);
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar_a), "r"(bq + bv) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)), "l"(qpos + (size_t)tile * ITILE * QPOS_W), "r"(bq), "r"(bar_a) : "memory");
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst + (size_t)ITILE * QPOS_W * sizeof(real))), "l"(qvel + (size_t)tile * ITILE * QVEL_W), "r"(bv), "r"(bar_a) : "memory");
  };
  if (threadIdx.x == 0) for (int s = 0; s < ISTAGES; ++s) { const int tile = blockIdx.x + s * gridDim.x; if (tile < ntiles) issue_load(s, tile); }
  for (int i = 0;; ++i) {
    const int tile = blockIdx.x + i * gridDim.x;
    if (tile >= ntiles) break;
    const int stage = i % ISTAGES; const uint32_t parity = (uint32_t)((i / ISTAGES) & 1), bar_a = smem_u32(&bar[stage]);
    asm volatile("{\n .reg .pred p;\n WAIT_%=:\n mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n @p bra DONE_%=;\n bra WAIT_%=;\n DONE_%=:\n}\n" ::"r"(bar_a), "r"(parity) : "memory");
    real *sq = reinterpret_cast<real *>(ibuf + (size_t)stage * itile_bytes<real>(QPOS_W, QVEL_W)); const real *sv = sq + ITILE * QPOS_W;
    const int cnt = min(ITILE, n - tile * ITILE);
    // scalar joints: lane = joint, warps stride over the tile's environments (a row's 36 entries sit in distinct banks);
    // ball joints: thread = (env, ball joint), dense, no divergence
    {
      const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
      if (lane < ns) { const int qa = sq_adr[lane], da = sd_adr[lane]; for (int e = wid; e < cnt; e += nw) sq[e * QPOS_W + qa] += h * sv[e * QVEL_W + da]; }
      for (int w = threadIdx.x; w < cnt * nb; w += blockDim.x) {
        const int e = w / nb, k = w - e * nb;
        real *q = sq + e * QPOS_W + bq_adr[k]; const real *v = sv + e * QVEL_W + bd_adr[k];
        real wv[3] = {v[0], v[1], v[2]}, qq[4] = {q[0], q[1], q[2], q[3]}, qr[4], s, c;
        const real ang = h * normalize3(wv);
        msincos(real(0.5) * ang, &s, &c); qr[0] = c; qr[1] = wv[0] * s; qr[2] = wv[1] * s; qr[3] = wv[2] * s;
        if (ang == 0) { qr[0] = 1; qr[1] = qr[2] = qr[3] = 0; }
        normalize4(qq); mul_quat(qq, qq, qr);
        q[0] = qq[0]; q[1] = qq[1]; q[2] = qq[2]; q[3] = qq[3];
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // generic-proxy writes -> visible to the bulk store
    __syncthreads();
    if (threadIdx.x == 0) {
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(qpos + (size_t)tile * ITILE * QPOS_W), "r"(smem_u32(sq)), "r"((uint32_t)(cnt * QPOS_W * sizeof(real))) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
      const int next = tile + ISTAGES * gridDim.x;
      if (next < ntiles) { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); issue_load(stage, next); }
    }
  }
  if (threadIdx.x == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
}

// rows of the selected environments <- one template row (masked reset / set_const)
template <typename T>
__global__ void fill_rows_kernel(T *__restrict__ dst, const T *__restrict__ row, int w, const unsigned char *__restrict__ mask, int n, int ncols) {
  const size_t total = (size_t)n * w;   // only the first ncols columns of a row are rewritten
  for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) { const size_t e = i / w; if ((!mask || mask[e]) && (int)(i - e * w) < ncols) dst[i] = row[i - e * w]; }
}

// ------------------------------------------------------------------ host side
// device-resident copy of every per-environment row array of a batch (cassie_state_t / cassie_batch_get_state); it owns its memory and carries its own
// sizes, so it can be copied, restored into any batch of the same shape and freed without the batch it was taken from
struct Snap {
  enum { R_QPOS, R_QVEL, R_QACC, R_CST, R_XFRC, R_OBS, R_DFILT, R_EST, R_AUX, R_APPL, NROWS };
  int device = 0, n = 0, esz = 4, qw = 0, vw = 0; bool has_est = false, has_aux = false, has_appl = false;   // has_appl: the applied-force rows
  void *rows[NROWS] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  bool has(int r) const { return !((r == R_EST && !has_est) || (r == R_AUX && !has_aux) || (r == R_APPL && !has_appl)); }   // the optional rows it holds
  // the frame rows [n][frame_list.size() / 2][FRAME_W] of the batch, with its frame list ((kind, id) pairs); restored only into a batch with the same list
  void *frames = nullptr; std::vector<int> frame_list;
  size_t frame_bytes() const { return (size_t)n * (frame_list.size() / 2) * FRAME_W * esz; }
  // the acceleration rows [n][acc_width(count)] of the batch (mjData's qacc and the cacc of its frames), if it had them; restored like the frame rows
  void *acc = nullptr;
  size_t acc_bytes() const { return (size_t)n * acc_width((int)(frame_list.size() / 2)) * esz; }
  int width(int r) const { const int w[NROWS] = {qw, vw, vw, CST_W, XFRC_W, OBS_W, DFILT_W, EST_W, AUX_W, APPLIED_W}; return w[r]; }
  int elem(int r) const { return r == R_DFILT ? 4 : (r == R_EST ? 8 : esz); }
  size_t bytes(int r) const { return (size_t)n * width(r) * elem(r); }
};
static void snap_delete(Snap *k) { if (!k) return; cudaSetDevice(k->device); for (int r = 0; r < Snap::NROWS; r++) cudaFree(k->rows[r]); cudaFree(k->frames); cudaFree(k->acc); delete k; }
static Snap *snap_new(int device, int n, int esz, int qw, int vw) {
  if (cudaSetDevice(device) != cudaSuccess) return nullptr;
  Snap *k = new Snap(); k->device = device; k->n = n; k->esz = esz; k->qw = qw; k->vw = vw;
  for (int r = 0; r < Snap::NROWS; r++) if (k->has(r) && cudaMalloc(&k->rows[r], k->bytes(r)) != cudaSuccess) { snap_delete(k); return nullptr; }
  return k;
}
static bool snap_clone_into(Snap *d, const Snap *k) {   // same shape required
  if (d->n != k->n || d->esz != k->esz || d->qw != k->qw || d->vw != k->vw || cudaSetDevice(d->device) != cudaSuccess) return false;
  d->has_est = k->has_est; d->has_aux = k->has_aux; d->has_appl = k->has_appl;
  for (int r = 0; r < Snap::NROWS; r++) {
    if (!k->has(r)) continue;
    if (!d->rows[r] && cudaMalloc(&d->rows[r], d->bytes(r)) != cudaSuccess) return false;
    if (cudaMemcpy(d->rows[r], k->rows[r], k->bytes(r), cudaMemcpyDefault) != cudaSuccess) return false;
  }
  if (d->frame_list != k->frame_list) { cudaFree(d->frames); cudaFree(d->acc); d->frames = d->acc = nullptr; d->frame_list = k->frame_list; if (k->frames && cudaMalloc(&d->frames, k->frame_bytes()) != cudaSuccess) return false; }
  if (k->frames && cudaMemcpy(d->frames, k->frames, k->frame_bytes(), cudaMemcpyDefault) != cudaSuccess) return false;
  if (!k->acc) { cudaFree(d->acc); d->acc = nullptr; }
  else if ((!d->acc && cudaMalloc(&d->acc, k->acc_bytes()) != cudaSuccess) || cudaMemcpy(d->acc, k->acc, k->acc_bytes(), cudaMemcpyDefault) != cudaSuccess) return false;
  return true;
}

struct BatchBase {
  virtual ~BatchBase() {}
  bool est_forces = false;   // fill toeForce / heelForce of state_out_t on the host (cassie_batch_enable_estimator_forces)
  bool est_filter = false;   // run the estimator's filters on the host, one per environment (cassie_batch_enable_estimator_filter; needs est_forces): the checker of the in-kernel estimator
  double aos_t[6] = {0, 0, 0, 0, 0, 0}; cudaEvent_t aos_ev[3] = {nullptr, nullptr, nullptr};   // [4] [5]: H2D and kernel milliseconds by CUDA events, only with CASSIE_B200_AOS_EVENTS set
  double aos_unused[1] = {0};   // accumulated seconds of the AoS entry point: host pack, device (copies + kernel, as waited for), host unpack; [3] calls
  bool est_auto = true;      // cassie_sim_step_pd_batch switches the in-kernel estimator on by itself (cassie_batch_enable_estimator_device(b, 0) clears this)
  std::vector<cassie::EstimatorFilter> est_state;
  void reset_estimator(const unsigned char *mask) { for (size_t e = 0; e < est_state.size(); e++) if (!mask || mask[e]) est_state[e].reset(); }
  HostModel hm; int n = 0, device = 0, precision = 0, wpb = 4; cudaStream_t stream = nullptr; bool own_stream = false; long launches = 0; bool debug = false;
  virtual bool init() = 0;
  virtual bool reset(const unsigned char *mask) = 0;
  virtual bool set_pd(const double *pd) = 0;
  virtual bool step(int nticks, int mode) = 0;
  virtual bool integrate() = 0;
  virtual bool get(const char *field, double *out) = 0;   // qpos[n][35] qvel[n][32] time[n] obs[n][64]
  virtual bool set(const char *field, const double *in) = 0;
  virtual bool set_xfrc(const double *xfrc, int body) = 0;
  virtual void *dev_ptr(const char *field) = 0;
  virtual bool get_counters(int *out) = 0;
  virtual int debug_dump(int env, double *out, int cnt) = 0;
  virtual bool step_pd_aos(const pd_in_t *pd_in, state_out_t *state_out, const double *radio) = 0;
  virtual bool set_hfield(const float *data, int n_terrains) = 0;
  virtual bool enable_aux(bool on) = 0;
  virtual bool enable_estimator_device(bool on) = 0;   // leg forces + filters inside the step kernel (extended instance), every 2 kHz tick
  virtual bool reset_estimator_device(const unsigned char *mask) = 0;
  virtual bool set_task_pd(const double *rows) = 0;   // [n][60] or null (off)
  virtual bool set_pd_gait(const double *amp, const double *freq, const double *phase) = 0;   // [n][10], [n], [n][10] or all null (off)
  virtual bool set_model_rows(const char *what, const double *rows, int width) = 0;   // per-env model constants (domain randomisation)
  virtual bool get_model_rows(const char *what, double *rows, int width) = 0;
  virtual bool set_const(const unsigned char *mask, bool reset_state) = 0;
  virtual bool has_aux() const = 0;
  // full dynamic state of every environment (cassie_get_state / cassie_set_state, src/cassiemujoco.c:3435-3452: mjData + the block objects +
  // cassie_out + encoder filters + torque delay line): device-resident snapshots, restore of a masked subset
  virtual Snap *snap_alloc() = 0;
  virtual bool snap_get(Snap *snap) = 0;
  virtual bool snap_set(const Snap *snap, const unsigned char *mask) = 0;
  // the reset bank: k start states gathered on the device from environments envs (null: 0 .. k - 1) of a snapshot of the same precision and model
  // (any size); k = 0 or a null snapshot drops it.  Checked before anything changes: a refused call keeps the old bank
  virtual bool set_reset_bank(const Snap *snap, const int *envs, int k) = 0;
  virtual int reset_bank_size() const = 0;
  // device-masked restore from the bank and device-masked mj_forward: enqueued on the batch's stream, no host synchronisation, copy or allocation
  virtual bool reset_where(const void *d_mask, const void *d_entry) = 0;
  virtual bool forward_where(const void *d_mask) = 0;
  // loop closure (loops.inl): the selected environments' qpos and qvel projected onto the connect equalities, one launch on the batch's stream; the
  // first call allocates the status rows [n][LOOP_SLOT].  get_loop_status copies them; any pointer may be null
  virtual bool close_loops(const void *d_mask, int max_iter, double tol) = 0;
  virtual bool get_loop_status(double *residual, int *iterations, double *vel_residual) = 0;
  // inverse kinematics (ik.inl): set_ik allocates the target and status rows (count 0 frees them); solve_ik is one launch on the batch's stream;
  // get_ik_status copies the status rows [n][IK_SLOT]
  virtual bool set_ik(const char *const *names, const int *kinds, const int *frames, const double *weights, int count) = 0;
  virtual bool solve_ik(const void *d_mask, int max_iter, double tol, int velocities) = 0;
  virtual bool get_ik_status(double *status) = 0;
  bool legacy = false;   // the batch of a cassie_sim_t: its host mirrors are pushed before every launch, so device-side resets are refused
  virtual bool copy_model_from(BatchBase *src) = 0;     // per-environment constants, height fields, timestep (mj_copyModel in cassie_sim_copy, :1083-1091)
  virtual bool rebuild_model() = 0;                     // after hm was edited (timestep, hold / release): rebuild and upload the constant block
  // per-environment placement of static planes / boxes (GEOM_ENV_W rows): pos / quat / size [n][3] / [n][4] / [n][3] or null (that part unchanged)
  virtual bool set_env_geom(int g, const double *pos, const double *quat, const double *size, const unsigned char *mask) = 0;
  virtual bool get_env_geom(int g, double *pos, double *quat, double *size) = 0;
  virtual bool clear_env_geoms() = 0;
  virtual bool shared_geom_changed(int g) = 0;          // after the shared placement of geom g was rebuilt: its slot in every row follows it
  // per-environment terrain: bank entry [n], height-field position [n][3] (in its body frame) and size [n][4]; NULL parts unchanged, only masked
  // environments change; checked as a whole before anything changes
  virtual bool set_env_hfield(const int *terrain, const double *pos, const double *size, const unsigned char *mask) = 0;
  virtual bool get_env_hfield(int *terrain, double *pos, double *size) = 0;
  virtual bool clear_env_hfield() = 0;
  virtual bool set_hfield_size(const double *size) = 0;   // the shared size; every environment's height-field position and size follow the shared ones
  // per-environment body offsets [n][nbody][3] (F_BP instances): only masked environments change; checked as a whole before anything changes
  virtual bool set_env_body_pos(const double *pos, const unsigned char *mask) = 0;
  virtual bool get_env_body_pos(double *pos) = 0;
  virtual bool clear_env_body_pos() = 0;
  // per-environment actuators (F_AC instances): ctrlrange [n][nu][2], rpm [n][nu], delay [n][nu], each may be null (kept); only masked environments
  // change; checked as a whole before anything changes
  virtual bool set_env_actuators(const double *ctrlrange, const double *rpm, const int *delay, const unsigned char *mask) = 0;
  virtual bool get_env_actuators(double *ctrlrange, double *rpm, int *delay) = 0;
  virtual bool clear_env_actuators() = 0;
  // per-environment mechanics (F_MC instances): inertia [n][nbody][3], armature [n][nv], stiffness and springref [n][njnt], each may be null (kept); only
  // masked environments change; checked as a whole before anything changes
  virtual bool set_env_mechanics(const double *inertia, const double *armature, const double *stiffness, const double *springref, const unsigned char *mask) = 0;
  virtual bool get_env_mechanics(double *inertia, double *armature, double *stiffness, double *springref) = 0;
  virtual bool clear_env_mechanics() = 0;
  // per-environment contact softness (F_CT instances): solref [n][ngeom][2], solimp [n][ngeom][5], solmix [n][ngeom], each may be null (kept); only
  // masked environments change; checked as a whole before anything changes
  virtual bool set_env_contact(const double *solref, const double *solimp, const double *solmix, const unsigned char *mask) = 0;
  virtual bool get_env_contact(double *solref, double *solimp, double *solmix) = 0;
  virtual bool clear_env_contact() = 0;
  // per-environment applied forces (F_XF instances; state): xfrc [n][nbody][6], qfrc [n][nv], either may be null (kept); only masked environments
  // change; checked as a whole before anything changes.  enable(false) drops the rows; clear_applied_xfrc zeroes the body wrenches of every environment
  virtual bool set_applied_forces(const double *xfrc, const double *qfrc, const unsigned char *mask) = 0;
  virtual bool get_applied_forces(double *xfrc, double *qfrc) = 0;
  virtual bool enable_applied_forces(bool on) = 0;
  virtual bool clear_applied_xfrc() = 0;
  // per-tick trace (F_TC instances; an output): k columns (source, column), the last max_ticks ticks of every step launch; k = 0 drops it.  Checked as a
  // whole before anything changes.  get copies [n][T][k]; trace_ticks is the number of slots the last step launch wrote
  virtual bool set_trace(const int *source, const int *column, int k, int max_ticks) = 0;
  virtual bool get_trace(double *out) = 0;
  virtual int trace_ticks() const = 0;
  virtual int trace_width() const = 0;   // T * k, 0 without a trace
  // contact lists (F_CL instances; an output): on allocates zeroed rows [n][CON_W], off frees them and returns the batch to the instance it ran before;
  // get copies [n][CON_W]
  virtual bool enable_contacts(bool on) = 0;
  virtual bool get_contacts(double *out) = 0;
  // sensor models (F_SN instances; a model input): encoder offset [n][16] and std [n][16], IMU mount [n][4], bias [n][6] (gyro, accelerometer) and std
  // [n][9] (orientation, gyro, accelerometer); null parts are kept, only masked environments change, checked as a whole before anything changes.  The
  // generator rows: key seed + i and counter 0 for the masked environments; get returns key and counter [n] each
  virtual bool set_env_sensors(const double *enc_offset, const double *enc_noise, const double *imu_quat, const double *imu_bias, const double *imu_noise, const unsigned char *mask) = 0;
  virtual bool get_env_sensors(double *enc_offset, double *enc_noise, double *imu_quat, double *imu_bias, double *imu_noise) = 0;
  virtual bool clear_env_sensors() = 0;
  virtual bool seed_sensors(unsigned long long seed, const unsigned char *mask) = 0;
  virtual bool get_sensor_rng(unsigned long long *seed, unsigned long long *counter) = 0;
  // the controller-stage state of every environment (views of the cst / dfilt rows): delay line [n][10][6], drive FIR taps [n][10][9], joint IIR
  // filters x [n][6][4] and y [n][6][3]; null parts are skipped, set changes masked environments only
  virtual bool get_actuator_state(double *torque_delay, int *drive_filter, double *joint_x, double *joint_y) = 0;
  virtual bool set_actuator_state(const double *torque_delay, const int *drive_filter, const double *joint_x, const double *joint_y, const unsigned char *mask) = 0;
  virtual bool set_frames(const char *const *names, const int *kinds, int count) = 0;   // frame rows [n][count][FRAME_W]; count 0: none
  virtual bool frame_jacobian(int frame, double *jacp, double *jacr) = 0;                 // [n][3][nv] each at the current state (launch mode 4); jacr may be null
  virtual bool dynamics() = 0;                                                            // one launch of mode 5 (asynchronous): the dynamics rows [n][DYN_W]
  virtual bool get_dynamics(double *M, double *bias, double *J_eq, double *eq_err, double *Icm) = 0;   // what the last mode-5 launch wrote; any pointer may be null
  bool dyn_done = false;                                // a mode-5 launch was enqueued since the rows were allocated
  // inverse dynamics (mode 6): qacc [n][nv] uploaded into the inverse-input rows [n][qvel width], or null: those rows as the caller left them on the
  // device; then one launch (asynchronous).  get_inverse: qfrc_inverse, qfrc_constraint [n][nv] and counts [n][3] of the last launch; any may be null
  virtual bool inverse(const double *qacc) = 0;
  virtual bool get_inverse(double *qfrc_inverse, double *qfrc_constraint, int *counts) = 0;
  bool inv_done = false;                                // a mode-6 launch was enqueued since the rows were allocated
  // acceleration rows [n][acc_width(count)]: allocated (zero) by enable_accelerations(true), filled by every step / forward launch, reallocated by set_frames
  virtual bool enable_accelerations(bool on) = 0;
  virtual bool get_accelerations(double *qacc, double *cacc) = 0;   // qacc [n][nv], cacc [n][count][6]; either may be null
  // terrain rays (raycast.inl): the table is checked as a whole before anything changes; k = 0 drops it.  The rows [n][k][RAY_SLOT] are allocated by
  // the first cast after a set and are a query result, not state
  virtual bool set_rays(const int *frame, const double *origin, const double *dir, const double *max_dist, int k) = 0;
  virtual bool raycast() = 0;                           // one launch (asynchronous) at the current qpos
  virtual bool get_rays(double *out) = 0;               // [n][k][RAY_SLOT] of the last cast
  int nray = 0; bool rays_done = false;                 // rays in the table; a cast was enqueued since the table was set
  // the depth cameras (camera.inl, camera_set.inl): a set of k <= CAM_MAX cameras with one image size and zfar, each mounted on a body; a set is checked as a whole
  // before anything changes, k = 0 drops it, and every set drops the depth, geom-id and per-environment mount rows.  The depth and geom-id rows
  // [n][k][height][width] are allocated by the first render after a set and are a query result, not state.  The mount rows [n][k][CAMENV_SLOT] are a
  // model input: allocated by set_env_cameras (holding the set's mounts), left alone by resets and snapshots
  struct Cameras { int k = 0, width = 0, height = 0, body[CAM_MAX] = {}; double pos[CAM_MAX][3] = {}, quat[CAM_MAX][4] = {}, fovy[CAM_MAX] = {}, zfar = 1; } cam;
  bool depth_done = false, geoms_done = false;          // a render was enqueued since the set (since the geom-id rows were enabled)
  bool cam_geoms = false;                               // renders write geom-id rows (cassie_batch_enable_camera_geoms)
  // k cameras: body [k], pos [k][3], quat [k][4] (normalised here), fovy [k]; indexed: refusals name the camera ("camera i: ...")
  virtual bool set_cameras(int k, const int *body, const double *pos, const double *quat, const double *fovy, int width, int height, double zfar,
                           const char *verb, bool indexed) = 0;
  virtual bool render_depth() = 0;                      // one launch (asynchronous) at the current qpos
  virtual bool get_depth(double *out) = 0;              // [n][k][height][width] of the last render
  // per-environment mounts: pos [n][k][3], quat [n][k][4], fovy [n][k], each may be null (kept); only masked environments change; checked as a whole
  // before anything changes
  virtual bool set_env_cameras(const double *pos, const double *quat, const double *fovy, const unsigned char *mask) = 0;
  virtual bool get_env_cameras(double *pos, double *quat, double *fovy) = 0;
  virtual bool clear_env_cameras() = 0;
  virtual bool enable_camera_geoms(bool on) = 0;
  virtual bool get_camera_geoms(int *out) = 0;          // [n][k][height][width] model geom ids of the last render, -1 where nothing is hit
  std::vector<int> frame_list;                          // (kind, id) per frame of the current frame table
  int nsub_override = 0;                                // > 0: physics sub-steps per control tick of the next launches (cassie_sim_step_pd_no2khz)
  bool sync() { CUDA_OK(cudaStreamSynchronize(stream)); return true; }
};

// the step instances' dynamic shared-memory limit is a property of the function, shared by every batch of the process: a batch raises it to its own
// launch size and never lowers it, so a smaller batch created later does not invalidate the launches of a larger one
static cudaError_t raise_smem_limit(const void *entry, int bytes) {
  cudaFuncAttributes fa; cudaError_t e = cudaFuncGetAttributes(&fa, entry);
  if (e != cudaSuccess || fa.maxDynamicSharedSizeBytes >= bytes) return e;
  return cudaFuncSetAttribute(entry, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
}

template <typename real> struct Batch : BatchBase {
  DevModel<real> *d_model = nullptr; EnvArrays<real> A{}; int QW = QPOS_W_MAIN, VW = QVEL_W_MAIN;
  real *d_iq = nullptr;   // inverse-input rows [n][VW]: the qacc of the next mode-6 launch, which passes them as its warm start
  real *d_idbg = nullptr, *d_icst = nullptr; int *d_icnt = nullptr;   // a mode-6 launch's stage dump [n][D_SIZE], controller state [n][CST_W], counters [n][8]
  struct LaunchCfg { int wpb = 1; size_t smem = 0; int resident_ctas = 1; } cfg[3];   // [0] plain instance, [1] extended instance, [2] plain + estimator
  int feat = F_ALL;   // model features (F_XB | F_HFIELD | F_BOX): selects the kernel instance
  std::vector<real> h_tmp;
  real *pin_pd = nullptr, *pin_obs = nullptr, *pin_task = nullptr;   // pinned staging for the AoS entry point
  real *dpin_pd = nullptr, *dpin_obs = nullptr;                      // the same buffers as the device sees them (mapped)
  static constexpr int AOS_MAXC = 4;
  cudaEvent_t aos_done[AOS_MAXC] = {}, aos_start = nullptr;            // the AoS entry point's chunk launches: completion events,
  cudaStream_t aos_stream[AOS_MAXC] = {};                              // their streams
  bool task_from_aos = false;   // the task-PD rows were created by the AoS entry point's forwarding (not by cassie_batch_set_task_pd)
  float *d_hfield = nullptr; unsigned char *d_mask = nullptr; DevModel<real> h_model_copy{}; int geom_dev[256]; void *d_row = nullptr;
  real *d_rtab = nullptr, *d_rays = nullptr;   // ray table (RT_HDR + nray RT_W) and the rows of the last cast
  real *d_depth = nullptr;                     // depth rows of the last render
  int *d_camgeom = nullptr;                    // geom-id rows of the last render (with cam_geoms)
  real *d_camenv = nullptr;                    // per-environment camera mounts [n][k][CAMENV_SLOT], allocated by the first cassie_batch_set_env_cameras
  std::vector<double> ce_host;                 // [n][k][CAMENV_SLOT] the mounts every environment sees while d_camenv exists (in double: what get returns)
  int *d_gtab = nullptr;                       // [MGT] the model geom of each device geom (-1: none): contact lists and camera geom ids, built on first use
  real *d_genv = nullptr;                  // A.genv: [n][GEOM_ENV_W] per-environment static-geom placement, allocated by the first per-environment placement
  std::vector<double> ge_host[MGS];        // per static slot touched by a per-environment placement: [n][10] pos 3, quat 4, size 3 in the geom's body frame
  int *d_terrain = nullptr;                // A.terrain: [n] per-environment bank entries, allocated by the first per-environment terrain (F_TR instances)
  std::vector<double> hf_host;             // [n][7] height-field position (in its body frame) 3, size 4 per environment; empty: the shared ones
  // the per-environment row blocks of env_rows.h: constant rows, body offsets, actuators, mechanics, contact softness, applied forces.  Each is [n][width]
  // reals held in its EnvArrays field; lent: the RowBlock bits of blocks lent for another one (env_rows.h)
  unsigned lent = 0;
  std::vector<double> bp_host;             // [n][nbody][3] the offsets every environment sees while A.bpos exists (in double: what get returns)
  std::vector<double> ac_host;             // [n][nu][4] lo, hi, rpm, delay every environment sees while A.act exists (in double: what get returns)
  std::vector<double> mc_host;             // [n][mech_host_w()] inertia, armature, stiffness, springref every environment sees while A.mech exists (in double)
  std::vector<double> ct_host;             // [n][ngeom][8] solref, solimp, solmix every environment sees while A.contact exists (in double: what get returns)
  int tc_ticks = 0;                        // slots the last step launch wrote into the trace rows (A.trace: [n][T][k], allocated by cassie_batch_set_trace)
  Snap *bank = nullptr;                    // the reset bank (cassie_batch_set_reset_bank): a snapshot of k entries
  real *d_loops = nullptr;                 // [n][LOOP_SLOT] status rows of cassie_batch_close_loops, allocated (zero) by its first call
  real *d_ikt = nullptr, *d_ik = nullptr;  // [n][IK_MAX][IK_TW] target rows and [n][IK_SLOT] status rows of the IK target list (cassie_batch_set_ik)
  int ik_n = 0;                            // the list: its targets' bodies, frames, poses in their bodies and weights
  std::vector<int> ik_body, ik_frame; std::vector<double> ik_pos, ik_quat, ik_w;
  ~Batch() override {
    snap_delete(bank);
    cudaSetDevice(device);
    cudaFree(d_ik); cudaFree(d_ikt); cudaFree(d_loops); cudaFree(d_rtab); cudaFree(d_rays); cudaFree(d_depth); cudaFree(d_camgeom); cudaFree(d_camenv); cudaFree(d_gtab); cudaFree(d_genv); cudaFree(d_terrain); for (int b = 0; b <= R_APP; b++) cudaFree(row(b)); cudaFree(A.trace.rows); cudaFree((void *)A.trace.cols); cudaFree(A.cl.rows); cudaFree((void *)A.sn.rows); cudaFree(A.sn.rng); cudaFree(A.frames); cudaFree((void *)A.ftab); cudaFree(A.jac); cudaFree(A.dyn); cudaFree(A.acc); cudaFree(A.inv); cudaFree(d_iq); cudaFree(d_idbg); cudaFree(d_icst); cudaFree(d_icnt);
    cudaFree(d_model); cudaFree(A.qpos); cudaFree(A.qvel); cudaFree(A.qacc_ws); cudaFree(A.cst); cudaFree(A.pd); cudaFree(A.xfrc); cudaFree(A.obs); cudaFree(A.dbg);
    cudaFree(A.dfilt); cudaFree(A.counters); cudaFree(A.qM); cudaFree(A.ticket); cudaFree(A.aux); cudaFree(A.task); cudaFree(A.gait); cudaFree(A.est); if (pin_task) cudaFreeHost(pin_task); cudaFree(d_mask); cudaFree(d_row);
    for (int i = 0; i < AOS_MAXC; i++) { if (aos_done[i]) cudaEventDestroy(aos_done[i]); if (aos_stream[i]) cudaStreamDestroy(aos_stream[i]); } if (aos_start) cudaEventDestroy(aos_start);
    if (pin_pd) cudaFreeHost(pin_pd); if (pin_obs) cudaFreeHost(pin_obs); if (d_hfield) cudaFree(d_hfield);
    if (own_stream && stream) cudaStreamDestroy(stream);
  }
  bool init() override {
    CUDA_OK(cudaSetDevice(device));
    DevModel<real> *hmodel = (DevModel<real> *)calloc(1, model_bytes<real>()); std::string err; BuildInfo info;
    if (!build_dev_model(hm, *hmodel, err, &info)) { free(hmodel); set_err(err); return false; }
    static bool noted = false;   // once per process
    if (info.unsupported_pairs && !noted) noted = true, fprintf(stderr, "cassie_b200: note: %d candidate geom pairs involve box/hfield geoms that this build does not collide (skipped)\n", info.unsupported_pairs);
    CUDA_OK(cudaMalloc(&d_model, model_bytes<real>()));
    CUDA_OK(cudaMemcpy(d_model, hmodel, model_bytes<real>(), cudaMemcpyHostToDevice));
    h_model_copy = *hmodel; memcpy(geom_dev, info.geom_dev, sizeof geom_dev);
    feat = hmodel->xb >= 0 ? F_XB : 0;   // which kernel instance this model needs (step_inst.cu)
    for (int p = 0; p < hmodel->npair; p++) { const int k = pair_kind(hmodel->pair_code[p]); if (k == PAIR_HFIELD_SPHERE || k == PAIR_HFIELD_CAPSULE) feat |= F_HFIELD; else if (k >= PAIR_PLANE_BOX) feat |= F_BOX; }
    const int hmodel_ystride = hmodel->ystride; QW = hmodel->qpos_w; VW = hmodel->qvel_w; A.qpos_w = QW; A.qvel_w = VW; A.ystride = hmodel_ystride; A.xb = hmodel->xb; free(hmodel);
    A.n = n; A.hfield = nullptr; A.n_terrain = 1; A.hfield_stride = 0; { const char *e = getenv("CASSIE_B200_SYNCMASK"); A.cta_sync = getenv("CASSIE_B200_NOSYNC") ? 0 : (e ? (atoi(e) & 127) : 10); }   // which of the five per-sub-step rendezvous are on
    if (hm.nhfield == 1 && !set_hfield(nullptr, 1)) return false;
    CUDA_OK(cudaMalloc(&A.qpos, sizeof(real) * n * QW)); CUDA_OK(cudaMalloc(&A.qvel, sizeof(real) * n * VW)); CUDA_OK(cudaMalloc(&A.qacc_ws, sizeof(real) * n * VW));
    CUDA_OK(cudaMalloc(&A.cst, sizeof(real) * n * CST_W)); CUDA_OK(cudaMalloc(&A.pd, sizeof(real) * n * PD_W)); CUDA_OK(cudaMalloc(&A.xfrc, sizeof(real) * n * XFRC_W));
    CUDA_OK(cudaMalloc(&A.obs, sizeof(real) * n * OBS_W)); CUDA_OK(cudaMalloc(&A.dfilt, sizeof(int) * n * DFILT_W)); CUDA_OK(cudaMalloc(&A.counters, sizeof(int) * n * 8)); CUDA_OK(cudaMalloc(&A.qM, sizeof(real) * n * 2 * NM_MAX)); CUDA_OK(cudaMalloc(&A.ticket, sizeof(int)));
    CUDA_OK(cudaMemset(A.pd, 0, sizeof(real) * n * PD_W)); CUDA_OK(cudaMemset(A.obs, 0, sizeof(real) * n * OBS_W)); CUDA_OK(cudaMemset(A.counters, 0, sizeof(int) * n * 8));
    if (debug) { CUDA_OK(cudaMalloc(&A.dbg, sizeof(real) * n * D_SIZE)); CUDA_OK(cudaMemset(A.dbg, 0, sizeof(real) * n * D_SIZE)); }
    CUDA_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking)); own_stream = true;
    // warps per CTA: maximise resident warps per SM over 1..4 CTAs per SM (each CTA carries its own copy of the model block); the two kernel
    // instances have different scratch sizes, hence their own launch shapes
    int dev_smem = 0, sm_smem = 0, sms = 0;
    CUDA_OK(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, device));
    CUDA_OK(cudaDeviceGetAttribute(&sm_smem, cudaDevAttrMaxSharedMemoryPerMultiprocessor, device));
    CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    for (int ext = 0; ext < 3; ++ext) {
      const long wb = (long)warp_bytes<real>(hmodel_ystride, ext == 1), mb = (long)model_bytes<real>() + 256;   // + static shared (mbarrier) and alignment slack
      const char *w = getenv("CASSIE_B200_WPB"); int k_sel = 1;
      if (w) { k_sel = atoi(w); const int kmax = (int)(((long)dev_smem - mb) / wb); if (k_sel > kmax) k_sel = kmax; }
      else {
        int best = 0, kk[5] = {0, 0, 0, 0, 0};
        for (int ctas = 4; ctas >= 1; --ctas) {
          long per_cta = (long)sm_smem / ctas - 1024; if (per_cta > dev_smem) per_cta = dev_smem;
          int k = (int)((per_cta - mb) / wb); if (k > 16) k = 16; if (k < 0) k = 0;
          kk[ctas] = k; if (k * ctas > best) best = k * ctas;
        }
        // the batch is worked off in rounds of (resident warps) environments: take the shape with the fewest rounds among those within 15 % of the best
        // residency; on a tie the fewest CTAs per SM -- with the static schedule nothing is refilled mid-round
        long best_rounds = -1;
        for (int ctas = 1; ctas <= 4; ++ctas) if (kk[ctas] >= 1 && kk[ctas] * ctas * 100 >= best * 85) {
          const long slots = (long)kk[ctas] * ctas * (sms > 0 ? sms : 1), rounds = (n + slots - 1) / slots;
          if (best_rounds < 0 || rounds < best_rounds) { best_rounds = rounds; k_sel = kk[ctas]; }
        }
      }
      if (k_sel < 1 || k_sel > 16 || (long)model_bytes<real>() + k_sel * wb > (long)dev_smem) { set_err("not enough shared memory per block"); return false; }
      if (!w && sms > 0) {   // balance the rounds: with one resident CTA per SM, n / sms environments per CTA are worked off in ceil(. / k) rounds of
                             // k; the smallest k with the same number of rounds leaves fewer warps contending in every round
        int ctas_per_sm = 1; { long per_cta = (long)sm_smem / 2 - 1024; if ((per_cta - mb) / wb >= k_sel) ctas_per_sm = 2; }
        if (ctas_per_sm == 1) { const double per_cta = (double)n / sms; const int rounds = (int)std::ceil(per_cta / k_sel); if (rounds >= 1) { int kb = (int)std::ceil(per_cta / rounds); if (kb < 1) kb = 1; if (kb < k_sel) k_sel = kb; } }
      }
      cfg[ext].wpb = k_sel; cfg[ext].smem = model_bytes<real>() + (size_t)k_sel * wb;
      int per_sm = 0;
      // every instance a launch of this kind can run for this model (the same scratch, the same shape): the one picked for the model's features
      // plus the optional features of each instance of the kind
      for (const StepInstance &si : STEP_INSTANCES) if (si.dbl == std::is_same<real, double>::value && si.kind == ext) {
        const StepChoice s = select_step<real>(ext, feat | (si.feat & ~F_ALL));
        if (s.kind == ext && s.index >= 0) CUDA_OK(raise_smem_limit(STEP_INSTANCES[s.index].entry(), (int)cfg[ext].smem));
      }
      CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, STEP_INSTANCES[select_step<real>(ext, feat).index].entry(), 32 * k_sel, cfg[ext].smem));
      cfg[ext].resident_ctas = per_sm * sms < 1 ? 1 : per_sm * sms;
    }
    wpb = cfg[0].wpb;
    return reset(nullptr);
  }
  bool reset(const unsigned char *mask) override {
    CUDA_OK(cudaSetDevice(device));
    std::vector<real> qpos(QPOS_W_XB), qvel(QVEL_W_XB), qa(QVEL_W_XB), cst(CST_W), xf(XFRC_W); std::vector<int> df(DFILT_W);
    init_env_rows(hm, qpos.data(), qvel.data(), qa.data(), cst.data(), df.data(), xf.data());
    if (!mask) {
      std::vector<real> buf((size_t)n * CST_W); std::vector<int> ibuf((size_t)n * DFILT_W, 0);
      auto fill = [&](real *dst, const std::vector<real> &row, int w) -> bool { for (int e = 0; e < n; e++) memcpy(&buf[(size_t)e * w], row.data(), sizeof(real) * w); CUDA_OK(cudaMemcpyAsync(dst, buf.data(), sizeof(real) * n * w, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream)); return true; };
      if (!fill(A.qpos, qpos, QW) || !fill(A.qvel, qvel, VW) || !fill(A.qacc_ws, qa, VW) || !fill(A.cst, cst, CST_W) || !fill(A.xfrc, xf, XFRC_W)) return false;
      if (A.applied) CUDA_OK(cudaMemsetAsync(row(R_APP), 0, sizeof(real) * n * APPLIED_W, stream));   // applied forces are state, as in mjData
      CUDA_OK(cudaMemcpyAsync(A.dfilt, ibuf.data(), sizeof(int) * n * DFILT_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
      return step(0, 1);
    }
    // masked reset: rewrite the selected rows, then mj_forward for exactly those environments
    if (!upload_mask(mask)) return false;
    if (!fill_masked(A.qpos, qpos.data(), QW) || !fill_masked(A.qvel, qvel.data(), VW) || !fill_masked(A.qacc_ws, qa.data(), VW) || !fill_masked(A.cst, cst.data(), CST_W) ||
        !fill_masked(A.xfrc, xf.data(), XFRC_W) || !fill_masked(A.dfilt, df.data(), DFILT_W)) return false;
    if (A.applied) { const std::vector<real> zero(APPLIED_W, real(0)); if (!fill_masked(row(R_APP), zero.data(), APPLIED_W)) return false; }
    return step_masked(1);
  }
  bool upload_mask(const unsigned char *mask) {
    if (!d_mask) CUDA_OK(cudaMalloc(&d_mask, n));
    CUDA_OK(cudaMemcpyAsync(d_mask, mask, n, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  template <typename T> bool fill_masked(T *dst, const T *row, int w, int ncols = 1 << 30) {   // uses d_mask
    if (!d_row) CUDA_OK(cudaMalloc(&d_row, 4096));
    CUDA_OK(cudaMemcpyAsync(d_row, row, sizeof(T) * w, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    fill_rows_kernel<T><<<256, 256, 0, stream>>>(dst, (const T *)d_row, w, d_mask, n, ncols);
    CUDA_OK(cudaGetLastError()); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  bool step_masked(int mode) { A.mask = d_mask; const bool ok = step(0, mode); A.mask = nullptr; return ok; }
  // ---- per-environment model constants (domain randomisation; reference setters src/cassiemujoco.c:1303-1436)
  bool ensure_cenv() {
    if (A.cenv) return true;
    CUDA_OK(cudaSetDevice(device));
    std::vector<real> row(CE_W), all((size_t)n * CE_W); init_cenv_row(h_model_copy, row.data(), hm, geom_dev);
    for (int e = 0; e < n; e++) memcpy(&all[(size_t)e * CE_W], row.data(), sizeof(real) * CE_W);
    CUDA_OK(cudaMalloc(&A.cenv, sizeof(real) * n * CE_W));
    CUDA_OK(cudaMemcpyAsync(A.cenv, all.data(), sizeof(real) * n * CE_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  // ---- the per-environment row blocks (env_rows.h): which exist, pull, push, drop and copy, and the rule's plans carried out
  static constexpr int ROW_W[R_APP + 1] = {CE_W, BP_W, ACT_W, MECH_W, CONTACT_W, APPLIED_W};
  real *row(int b) const { const void *p[R_APP + 1] = {A.cenv, A.bpos, A.act, A.mech, A.contact, A.applied}; return (real *)p[b]; }
  void publish(int b, real *r) {
    switch (b) { case R_CENV: A.cenv = r; break; case R_BPOS: A.bpos = r; break; case R_ACT: A.act = r; break; case R_MECH: A.mech = r; break; case R_CT: A.contact = r; break; default: A.applied = r; }
  }
  std::vector<double> *mirror(int b) { std::vector<double> *m[R_APP + 1] = {nullptr, &bp_host, &ac_host, &mc_host, &ct_host, nullptr}; return m[b]; }
  RowState row_state() const {
    const void *p[R_N] = {A.cenv, A.bpos, A.act, A.mech, A.contact, A.applied, A.trace.rows, A.cl.rows, A.sn.rows};
    RowState s; s.lent = lent;
    for (int b = 0; b < R_N; b++) if (p[b]) s.have |= 1u << b;
    return s;
  }
  bool pull(int b, std::vector<real> &all) {   // the device rows (zero without rows)
    all.assign((size_t)n * ROW_W[b], real(0));
    if (!row(b)) return true;
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(all.data(), row(b), sizeof(real) * n * ROW_W[b], cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  bool alloc_rows(int b) { real *r = nullptr; if (!row(b)) { CUDA_OK(cudaMalloc(&r, sizeof(real) * n * ROW_W[b])); publish(b, r); } return true; }
  bool push(int b, const std::vector<real> &all) {
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a launch in flight reads the rows
    if (!alloc_rows(b)) return false;
    CUDA_OK(cudaMemcpy(row(b), all.data(), sizeof(real) * n * ROW_W[b], cudaMemcpyHostToDevice));
    return b != R_BPOS || put_reach();
  }
  bool drop(int b) {
    if (mirror(b)) mirror(b)->clear();
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a launch in flight reads the rows
    CUDA_OK(cudaFree(row(b))); publish(b, nullptr);
    return b != R_BPOS || rebuild_model();   // the block's robot_reach is the model's again
  }
  bool copy_rows(int b, Batch *src) {   // the source's rows as its environments run with them, and its mirror
    if (mirror(b)) *mirror(b) = *src->mirror(b);
    CUDA_OK(cudaStreamSynchronize(src->stream)); CUDA_OK(cudaStreamSynchronize(stream));
    if (!alloc_rows(b)) return false;
    CUDA_OK(cudaMemcpy(row(b), src->row(b), sizeof(real) * n * ROW_W[b], cudaMemcpyDeviceToDevice));
    return b != R_BPOS || put_reach();
  }
  bool put_model(int b) {   // the block's rows holding the model's values (applied forces: zero), allocated where absent
    std::vector<real> all;
    switch (b) {
      case R_CENV: return ensure_cenv();
      case R_BPOS: model_bpos_rows(); return put_bpos();
      case R_ACT: model_act_rows(all); break;
      case R_MECH: model_mech_rows(all); break;
      case R_CT: model_ct_rows(all); break;
      default: all.assign((size_t)n * APPLIED_W, real(0));
    }
    return push(b, all);
  }
  bool run(const RowPlan &p) {
    for (int i = 0; i < p.n; i++) if (!(p.step[i].op == ROW_DROP ? drop(p.step[i].block) : put_model(p.step[i].block))) return false;
    return true;
  }
  bool rows_rule(void (*rule)(RowState &, RowPlan &, int), int b) { RowState s = row_state(); RowPlan p; rule(s, p, b); lent = s.lent; return run(p); }
  int cenv_slot(const char *what, int i, int &width) const { return cassie::cenv_slot(hm, h_model_copy.nv, geom_dev, what, i, width); }
  bool set_model_rows(const char *what, const double *rows, int width) override {
    int w = 0; cenv_slot(what, 0, w);
    if (w < 0 || w != width) { set_err(std::string("set_model_rows: unknown array or wrong width for ") + what); return false; }
    if (!strcmp(what, "body_ipos") && h_model_copy.xb >= 0) for (int e = 0; e < n; e++) for (int k = 0; k < 3; k++)
      if (rows[(size_t)e * w + 3 * h_model_copy.xb + k] != hm.body_ipos[3 * h_model_copy.xb + k]) { set_err("body_ipos of the extra free body cannot be changed (its inertial frame must stay its body frame)"); return false; }
    if (!ensure_cenv() || !rows_rule(own, R_CENV)) return false;
    std::vector<real> all((size_t)n * CE_W);
    CUDA_OK(cudaMemcpyAsync(all.data(), A.cenv, sizeof(real) * n * CE_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) for (int i = 0; i < w; i++) { int ww; const int sl = cenv_slot(what, i, ww); if (sl >= 0) all[(size_t)e * CE_W + sl] = (real)rows[(size_t)e * w + i]; }
    CUDA_OK(cudaMemcpyAsync(A.cenv, all.data(), sizeof(real) * n * CE_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  bool get_model_rows(const char *what, double *rows, int width) override {
    int w = 0; cenv_slot(what, 0, w);
    if (w < 0 || w != width) { set_err(std::string("get_model_rows: unknown array or wrong width for ") + what); return false; }
    if (!ensure_cenv()) return false;
    std::vector<real> all((size_t)n * CE_W);
    CUDA_OK(cudaMemcpyAsync(all.data(), A.cenv, sizeof(real) * n * CE_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    const std::vector<double> *src = !strcmp(what, "geom_friction") ? &hm.geom_friction : nullptr;
    for (int e = 0; e < n; e++) for (int i = 0; i < w; i++) { int ww; const int sl = cenv_slot(what, i, ww); rows[(size_t)e * w + i] = sl >= 0 ? (double)all[(size_t)e * CE_W + sl] : (src ? (*src)[i] : 0.0); }
    return true;
  }
  // mj_setConst for the selected environments on the device (mode 3), optionally followed by the state reset cassie_sim_set_const performs
  bool set_const(const unsigned char *mask, bool reset_state) override {
    if (!ensure_cenv()) return false;
    std::vector<unsigned char> ones; if (!mask) { ones.assign(n, 1); mask = ones.data(); }
    if (!upload_mask(mask) || !step_masked(3)) return false;
    if (!reset_state) return sync();
    // src/cassiemujoco.c:955-971: qpos <- the init constants, qvel <- 0, time <- 0, mj_forward (filters, delay line, cassie_out keep their values)
    std::vector<real> qpos(QPOS_W_XB), qvel(QVEL_W_XB), qa(QVEL_W_XB), cst(CST_W), xf(XFRC_W); std::vector<int> df(DFILT_W);
    init_env_rows(hm, qpos.data(), qvel.data(), qa.data(), cst.data(), df.data(), xf.data());
    if (!fill_masked(A.qpos, qpos.data(), QW, 35) || !fill_masked(A.qvel, qvel.data(), VW)) return false;   // the reference copies 35 qpos entries (:967): an extra free body keeps its pose
    { std::vector<real> all((size_t)n * CST_W);
      CUDA_OK(cudaMemcpyAsync(all.data(), A.cst, sizeof(real) * n * CST_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
      for (int e = 0; e < n; e++) if (mask[e]) all[(size_t)e * CST_W + CS_TIME] = 0;
      CUDA_OK(cudaMemcpyAsync(A.cst, all.data(), sizeof(real) * n * CST_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream)); }
    return step_masked(1) && sync();
  }
  bool set_pd(const double *pd) override {
    h_tmp.resize((size_t)n * PD_W);
    for (size_t i = 0; i < (size_t)n * PD_W; i++) h_tmp[i] = (real)pd[i];
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(A.pd, h_tmp.data(), sizeof(real) * n * PD_W, cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaStreamSynchronize(stream));   // h_tmp is pageable and reused
    return true;
  }
  // cassie_sim_step_pd for every env with host AoS buffers: pack pd_in_t[] -> pinned rows -> H2D, one tick, D2H rows -> state_out_t[]
  bool step_pd_aos(const pd_in_t *pd_in, state_out_t *state_out, const double *radio) override {
    CUDA_OK(cudaSetDevice(device));
    static const int aos_threads = aos_thread_count();
    static const bool aos_events = getenv("CASSIE_B200_AOS_EVENTS") != nullptr;
    static const bool aos_obs_dma = [] { const char *e = getenv("CASSIE_B200_AOS_OBS_DMA"); return e && atoi(e) != 0; }();
    static const int aos_chunks = [] { const char *e = getenv("CASSIE_B200_AOS_CHUNKS"); int t = e ? atoi(e) : 2; return t < 1 ? 1 : (t > AOS_MAXC ? AOS_MAXC : t); }();   // launches per call for batches of up to two rounds
    if (!pin_pd) {   // pinned AND mapped: the step kernel itself writes the observation rows into pin_obs
      CUDA_OK(cudaHostAlloc(&pin_pd, sizeof(real) * n * PD_W, cudaHostAllocMapped)); CUDA_OK(cudaHostAlloc(&pin_obs, sizeof(real) * n * OBS_W, cudaHostAllocMapped));
      CUDA_OK(cudaHostGetDevicePointer(&dpin_pd, pin_pd, 0)); CUDA_OK(cudaHostGetDevicePointer(&dpin_obs, pin_obs, 0));
      for (int i = 0; i < AOS_MAXC; i++) { CUDA_OK(cudaEventCreateWithFlags(&aos_done[i], cudaEventDisableTiming)); CUDA_OK(cudaStreamCreateWithFlags(&aos_stream[i], cudaStreamNonBlocking)); }
      CUDA_OK(cudaEventCreateWithFlags(&aos_start, cudaEventDisableTiming));
    }
    auto now = [] { return std::chrono::steady_clock::now(); };
    auto sec = [](std::chrono::steady_clock::time_point a, std::chrono::steady_clock::time_point b) { return std::chrono::duration<double>(b - a).count(); };
    double t_pack = 0, t_wait = 0, t_unpack = 0;
    auto tq = now();
    // taskPd branch of pd_in_t: task rows are uploaded only while some environment uses that branch.  While task rows exist, the whole batch is
    // scanned before the first launch (and the rows are dropped again when no environment uses them); otherwise -- the common case, motor PD only --
    // the scan rides along with the chunks' pack loops, and the first chunk that finds a task entry installs the rows for itself and the later chunks
    // (the earlier chunks, by their own scan, had none).
    auto uses_task = [](const pd_in_t &u) { int any = 0; const pd_task_in_t *t[2] = {&u.leftLeg.taskPd, &u.rightLeg.taskPd};
      for (int sd = 0; sd < 2; sd++) for (int k = 0; k < 6; k++) any |= (t[sd]->torque[k] != 0 || t[sd]->pGain[k] != 0 || t[sd]->dGain[k] != 0); return any; };
    auto install_task_rows = [&](cudaStream_t on) -> bool {
      if (!pin_task) CUDA_OK(cudaMallocHost(&pin_task, sizeof(real) * n * TASK_W));
      if (!A.task) { CUDA_OK(cudaMalloc(&A.task, sizeof(real) * n * TASK_W)); task_from_aos = true; }
#pragma omp parallel for schedule(static) num_threads(aos_threads) if (n >= 512)
      for (int e = 0; e < n; e++) { real *row = pin_task + (size_t)e * TASK_W;
        for (int sd = 0; sd < 2; sd++) { const pd_task_in_t *t = sd ? &pd_in[e].rightLeg.taskPd : &pd_in[e].leftLeg.taskPd; real *r = row + 30 * sd;
          for (int k = 0; k < 6; k++) { r[k] = (real)t->torque[k]; r[6 + k] = (real)t->pTarget[k]; r[12 + k] = (real)t->dTarget[k]; r[18 + k] = (real)t->pGain[k]; r[24 + k] = (real)t->dGain[k]; } }
        for (int i = 60; i < TASK_W; i++) row[i] = 0; }
      CUDA_OK(cudaMemcpyAsync(A.task, pin_task, sizeof(real) * n * TASK_W, cudaMemcpyHostToDevice, on));
      return true; };
    bool scan_in_chunks = (A.task == nullptr);
    if (!scan_in_chunks) {
      int any = 0;
#pragma omp parallel for schedule(static) num_threads(aos_threads) reduction(| : any) if (n >= 512)
      for (int e = 0; e < n; e++) any |= uses_task(pd_in[e]);
      if (any) { if (!install_task_rows(stream)) return false; }
      else if (task_from_aos) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(A.task)); A.task = nullptr; task_from_aos = false; }   // rows installed with cassie_batch_set_task_pd stay
    }
    // cassie_sim_step_pd runs state_output_step in every call (src/cassiemujoco.c:1156): so does the batched entry point, inside the kernel,
    // from the first call that asks for state_out_t rows (unless the caller switched it off or runs the host-side checker instead)
    if (state_out && est_auto && !A.est && !est_filter && !enable_estimator_device(true)) return false;
    if (est_filter && est_state.size() != (size_t)n) est_state.assign((size_t)n, cassie::EstimatorFilter());
    const bool dev_est = A.est != nullptr;   // the estimator runs inside the kernel: its outputs are columns of the observation row
    // The batch is stepped as up to AOS_MAXC independent launches ("chunks") on their own streams: the host packs chunk c + 1 while chunk c is copied in
    // and stepping, and unpacks chunk c while the later ones are stepping; the kernels of consecutive chunks overlap at their edges (a chunk's CTAs start
    // on the SMs the previous chunk's CTAs have left, while its last observation rows are still draining over PCIe).  Chunks are whole rounds of the
    // resident warps when the batch is worked off in more than two rounds, equal parts otherwise.
    const int inst = (A.cenv || A.aux || A.task || A.frames || A.acc || (A.dbg && !DBG_IN_ALL_INSTANCES)) ? 1 : (A.est ? 2 : 0), slots = cfg[inst].resident_ctas * cfg[inst].wpb;
    int nchunk = 1, c0[AOS_MAXC + 1] = {0};
    if (state_out && n >= 1024 && aos_chunks > 1) {
      if (n <= 2 * slots) { nchunk = aos_chunks; for (int c = 1; c < nchunk; c++) c0[c] = (int)((size_t)n * c / nchunk + 31) / 32 * 32; }
      else { const int rounds = (n + slots - 1) / slots; nchunk = rounds < AOS_MAXC ? rounds : AOS_MAXC; const int per = (rounds + nchunk - 1) / nchunk * slots;
        for (int c = 1; c < nchunk; c++) c0[c] = per * c < n ? per * c : n; }
    }
    c0[nchunk] = n;
    CUDA_OK(cudaEventRecord(aos_start, stream));   // everything enqueued on the batch's stream so far happens before the chunks
    t_pack += sec(tq, now());
    for (int c = 0; c < nchunk; c++) {
      const int e0 = c0[c], e1 = c0[c + 1], cnt = e1 - e0; if (cnt <= 0) { CUDA_OK(cudaEventRecord(aos_done[c], stream)); continue; }
      tq = now();
      int any_task = 0;
#pragma omp parallel for schedule(static) num_threads(aos_threads) reduction(| : any_task) if (n >= 512)
      for (int e = e0; e < e1; e++) {
        real *row = pin_pd + (size_t)e * PD_W; const pd_in_t *u = pd_in + e;
        for (int i = 0; i < 10; i++) {
          const pd_motor_in_t *p = i < 5 ? &u->leftLeg.motorPd : &u->rightLeg.motorPd; const int k = i % 5;
          row[i] = (real)p->torque[k]; row[10 + i] = (real)p->pTarget[k]; row[20 + i] = (real)p->dTarget[k]; row[30 + i] = (real)p->pGain[k]; row[40 + i] = (real)p->dGain[k];
        }
        row[50] = row[51] = 0;
        if (scan_in_chunks) any_task |= uses_task(*u);
      }
      const size_t off = (size_t)e0 * PD_W; cudaStream_t cs = nchunk > 1 ? aos_stream[c] : stream;
      if (nchunk > 1) CUDA_OK(cudaStreamWaitEvent(cs, aos_start, 0));
      if (any_task) {   // first task entry of this call: rows for the whole batch, in place before this chunk's (and every later chunk's) launch
        if (!install_task_rows(cs)) return false;
        CUDA_OK(cudaStreamSynchronize(cs)); scan_in_chunks = false;
      }
      t_pack += sec(tq, now());
      if (aos_events && c == 0) { if (!aos_ev[0]) for (int i = 0; i < 3; i++) CUDA_OK(cudaEventCreate(&aos_ev[i])); CUDA_OK(cudaEventRecord(aos_ev[0], cs)); }
      CUDA_OK(cudaMemcpyAsync(A.pd + off, pin_pd + off, sizeof(real) * cnt * PD_W, cudaMemcpyHostToDevice, cs));   // one DMA per launch: a burst of small PCIe reads from every warp at kernel start measured no faster
      if (aos_events && c == 0) CUDA_OK(cudaEventRecord(aos_ev[1], cs));
      A.pd_host = nullptr; A.obs_host = (state_out && !aos_obs_dma) ? dpin_obs : nullptr;   // observation rows return by zero-copy stores as each environment finishes ...
      const bool launched = step_range(1, 0, e0, cnt, cs);
      A.obs_host = nullptr;
      if (!launched) return false;
      if (state_out && aos_obs_dma) CUDA_OK(cudaMemcpyAsync(pin_obs + (size_t)e0 * OBS_W, A.obs + (size_t)e0 * OBS_W, sizeof(real) * cnt * OBS_W, cudaMemcpyDeviceToHost, cs));   // ... or by one DMA per chunk
      CUDA_OK(cudaEventRecord(aos_done[c], cs));
      if (nchunk > 1) CUDA_OK(cudaStreamWaitEvent(stream, aos_done[c], 0));   // later work on the batch's stream sees the stepped rows
      if (aos_events && c == nchunk - 1) CUDA_OK(cudaEventRecord(aos_ev[2], cs));
    }
    if (!state_out) return sync();
    for (int c = 0; c < nchunk; c++) {
      tq = now();
      CUDA_OK(cudaEventSynchronize(aos_done[c]));
      t_wait += sec(tq, now()); tq = now();
#pragma omp parallel for schedule(static) num_threads(aos_threads) if (n >= 512)
      for (int e = c0[c]; e < c0[c + 1]; e++) {
      // every field of state_out_t is written exactly once (no memset pass): what the reference's block never writes (externalMoment,
      // terrain.slope, battery.current) is zero, as in a freshly set-up state_output_t
      const real *o = pin_obs + (size_t)e * OBS_W; state_out_t *y = state_out + e; const real *eo = o + OB_EST_OUT;
      for (int i = 0; i < 3; i++) { y->pelvis.position[i] = dev_est ? (double)eo[EO_POS + i] : 0.0; y->pelvis.translationalVelocity[i] = dev_est ? (double)eo[EO_VEL + i] : 0.0;
                                    y->pelvis.externalForce[i] = dev_est ? (double)eo[EO_EXTF + i] : 0.0; y->pelvis.externalMoment[i] = 0;
                                    y->pelvis.rotationalVelocity[i] = o[OB_GYRO + i]; y->pelvis.translationalAcceleration[i] = o[OB_EST_ACC + i]; }
      for (int i = 0; i < 4; i++) y->pelvis.orientation[i] = o[OB_EST_QUAT + i];
      y->terrain.height = dev_est ? (double)eo[EO_TERRAIN] : 0.0; y->terrain.slope[0] = y->terrain.slope[1] = 0;
      for (int i = 0; i < 10; i++) { y->motor.position[i] = o[OB_MPOS + i]; y->motor.velocity[i] = o[OB_MVEL + i]; y->motor.torque[i] = o[OB_MTORQUE + i]; }
      for (int i = 0; i < 6; i++) { y->joint.position[i] = o[OB_JPOS + i]; y->joint.velocity[i] = o[OB_JVEL + i]; }
      for (int sd = 0; sd < 2; sd++) {   // decoded estimator: foot pose (pelvis frame), velocities (foot frame), toe / heel force
        state_foot_out_t *f = sd ? &y->rightFoot : &y->leftFoot; const real *fo = o + OB_FOOT + 13 * sd;
        for (int i = 0; i < 3; i++) { f->position[i] = fo[i]; f->footRotationalVelocity[i] = fo[7 + i]; f->footTranslationalVelocity[i] = fo[10 + i]; }
        for (int i = 0; i < 4; i++) f->orientation[i] = fo[3 + i];
        if (est_forces || est_filter) {   // host-side checker path (cassie_batch_enable_estimator_forces / _filter): the same functions the kernel runs
          const double ang[7] = {o[OB_MPOS + 5 * sd], o[OB_MPOS + 5 * sd + 1], o[OB_MPOS + 5 * sd + 2], o[OB_MPOS + 5 * sd + 3], o[OB_JPOS + 3 * sd], o[OB_JPOS + 3 * sd + 1], o[OB_MPOS + 5 * sd + 4]};
          const double qd[4] = {o[OB_QUAT], o[OB_QUAT + 1], o[OB_QUAT + 2], o[OB_QUAT + 3]};
          estimator_leg_force(sd, ang, qd, f->toeForce);
        } else for (int i = 0; i < 3; i++) f->toeForce[i] = dev_est ? (double)eo[EO_TOE + 3 * sd + i] : 0.0;
        for (int i = 0; i < 3; i++) f->heelForce[i] = f->toeForce[i];
      }
      if (est_filter) {   // host-side checker path: one 2 kHz filter call per step_pd call, overwrites the four filtered outputs
        cassie::EstimatorFilter &f = est_state[(size_t)e];
        f.step(y->pelvis.orientation, y->leftFoot.position, y->rightFoot.position, y->leftFoot.toeForce[2] + y->leftFoot.heelForce[2],
               y->rightFoot.toeForce[2] + y->rightFoot.heelForce[2], y->pelvis.translationalAcceleration,
               y->pelvis.position, y->pelvis.translationalVelocity, y->pelvis.externalForce, &y->terrain.height);
      }
      for (int i = 0; i < 16; i++) y->radio.channel[i] = radio[(size_t)e * 16 + i];
      memset(&y->radio.signalGood, 0, sizeof(double)); y->radio.signalGood = true;   // the bool and its padding
      y->battery.stateOfCharge = 1; y->battery.current = 0;
      }
      t_unpack += sec(tq, now());
    }
    aos_t[0] += t_pack; aos_t[1] += t_wait; aos_t[2] += t_unpack; aos_t[3] += 1;
    if (aos_events) { float a = 0, b = 0; cudaEventElapsedTime(&a, aos_ev[0], aos_ev[1]); cudaEventElapsedTime(&b, aos_ev[1], aos_ev[2]); aos_t[4] += a; aos_t[5] += b; }
    return true;
  }
  // K terrains of nrow*ncol normalised elevations; environment e stands on terrain e % K (cassie_sim_set_hfielddata, src/cassiemujoco.c:2076-2080)
  bool set_hfield(const float *data, int n_terrains) override {
    if (hm.nhfield != 1 || n_terrains < 1) { set_err("this model has no height field"); return false; }
    CUDA_OK(cudaSetDevice(device));
    const size_t cells = (size_t)hm.hfield_nrow[0] * hm.hfield_ncol[0];
    CUDA_OK(cudaStreamSynchronize(stream));
    if (d_hfield) CUDA_OK(cudaFree(d_hfield));
    CUDA_OK(cudaMalloc(&d_hfield, sizeof(float) * cells * n_terrains));
    if (data) CUDA_OK(cudaMemcpy(d_hfield, data, sizeof(float) * cells * n_terrains, cudaMemcpyHostToDevice));
    else CUDA_OK(cudaMemset(d_hfield, 0, sizeof(float) * cells * n_terrains));
    A.hfield = d_hfield; A.n_terrain = n_terrains; A.hfield_stride = cells;
    return true;
  }
  // derived-quantity rows [n][AUX_W]: allocated on first use; while present every launch fills them (a few percent of a step)
  bool enable_aux(bool on) override {
    if (!on && A.aux && ((A.trace.need >> TC_AUX) & 1)) { set_err("cassie_batch_enable_aux: a traced column reads the derived-quantity rows (cassie_batch_set_trace)"); return false; }
    CUDA_OK(cudaSetDevice(device));
    if (on && !A.aux) { CUDA_OK(cudaMalloc(&A.aux, sizeof(real) * n * AUX_W)); CUDA_OK(cudaMemsetAsync(A.aux, 0, sizeof(real) * n * AUX_W, stream)); }
    if (!on && A.aux) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(A.aux)); A.aux = nullptr; }
    return true;
  }
  bool has_aux() const override { return A.aux != nullptr; }
  bool enable_estimator_device(bool on) override {
    CUDA_OK(cudaSetDevice(device));
    if (on && !A.est) {
      CUDA_OK(cudaMalloc(&A.est, sizeof(double) * n * EST_W));
      CUDA_OK(cudaMemsetAsync(A.est, 0, sizeof(double) * n * EST_W, stream));
    }
    if (!on && A.est) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(A.est)); A.est = nullptr;
                        CUDA_OK(cudaMemset2DAsync(A.obs + OB_EST_OUT, sizeof(real) * OBS_W, 0, sizeof(real) * EO_W, n, stream)); }   // its columns of the observation row read zero again
    return true;
  }
  bool reset_estimator_device(const unsigned char *mask) override {   // started flag (and everything else) back to zero: the filters start again at the next tick
    if (!A.est) return true;
    CUDA_OK(cudaSetDevice(device));
    if (!mask) { CUDA_OK(cudaMemsetAsync(A.est, 0, sizeof(double) * n * EST_W, stream)); return true; }
    if (!upload_mask(mask)) return false;
    const std::vector<double> zero(EST_W, 0.0);
    return fill_masked(A.est, zero.data(), EST_W);
  }
  // task-space PD rows (pd_in_t taskPd of both legs); NULL switches the branch off again
  bool set_task_pd(const double *rows) override {
    CUDA_OK(cudaSetDevice(device));
    task_from_aos = false;   // the caller owns the rows from here on: the AoS entry point no longer drops them
    if (!rows) { if (A.task) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(A.task)); A.task = nullptr; } return true; }
    if (!A.task) CUDA_OK(cudaMalloc(&A.task, sizeof(real) * n * TASK_W));
    h_tmp.assign((size_t)n * TASK_W, 0);
    for (int e = 0; e < n; e++) for (int i = 0; i < 60; i++) h_tmp[(size_t)e * TASK_W + i] = (real)rows[(size_t)e * 60 + i];
    CUDA_OK(cudaMemcpyAsync(A.task, h_tmp.data(), sizeof(real) * n * TASK_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  // ---- snapshots (the Snap object owns its device memory and knows its own sizes: it may outlive this batch)
  Snap *snap_alloc() override { Snap *k = snap_new(device, n, (int)sizeof(real), QW, VW); if (!k) set_err("snapshot: out of device memory"); return k; }
  bool snap_compatible(const Snap *k) { if (k && k->n == n && k->esz == (int)sizeof(real) && k->qw == QW && k->vw == VW) return true; set_err("snapshot: taken from a batch of another size, precision or model"); return false; }
  void *snap_src(int r) { void *t[Snap::NROWS] = {A.qpos, A.qvel, A.qacc_ws, A.cst, A.xfrc, A.obs, A.dfilt, A.est, A.aux, row(R_APP)}; return t[r]; }
  bool snap_get(Snap *k) override {
    if (!snap_compatible(k)) return false;
    CUDA_OK(cudaSetDevice(device));
    k->has_est = A.est != nullptr; k->has_aux = A.aux != nullptr; k->has_appl = A.applied != nullptr;
    for (int r = 0; r < Snap::NROWS; r++) {
      if (!k->has(r)) continue;
      if (!k->rows[r]) CUDA_OK(cudaMalloc(&k->rows[r], k->bytes(r)));
      CUDA_OK(cudaMemcpyAsync(k->rows[r], snap_src(r), k->bytes(r), cudaMemcpyDeviceToDevice, stream));
    }
    if (k->frame_list != frame_list) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(k->frames)); CUDA_OK(cudaFree(k->acc)); k->frames = k->acc = nullptr; k->frame_list = frame_list; if (A.frames) CUDA_OK(cudaMalloc(&k->frames, k->frame_bytes())); }
    if (A.frames) CUDA_OK(cudaMemcpyAsync(k->frames, A.frames, k->frame_bytes(), cudaMemcpyDeviceToDevice, stream));
    if (A.acc) { if (!k->acc) CUDA_OK(cudaMalloc(&k->acc, k->acc_bytes())); CUDA_OK(cudaMemcpyAsync(k->acc, A.acc, k->acc_bytes(), cudaMemcpyDeviceToDevice, stream)); }
    else if (k->acc) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(k->acc)); k->acc = nullptr; }
    return sync();
  }
  bool snap_set(const Snap *k, const unsigned char *mask) override {
    if (!snap_compatible(k)) return false;
    CUDA_OK(cudaSetDevice(device));
    if (mask && !upload_mask(mask)) return false;
    if (k->has_est && !A.est && !enable_estimator_device(true)) return false;   // optional rows the snapshot has are allocated where the batch lacks them
    if (k->has_appl && !A.applied && !enable_applied_forces(true)) return false;
    if (mask) return restore_rows(k, d_mask, nullptr) && sync();   // one launch: the snapshot as a bank of n entries, environment e taking entry e
    if (!k->has_est && A.est && !reset_estimator_device(nullptr)) return false;   // the snapshot was taken before the estimator ran: it starts afresh
    if (!k->has_appl && A.applied) CUDA_OK(cudaMemsetAsync(row(R_APP), 0, sizeof(real) * n * APPLIED_W, stream));   // likewise the applied forces: zeroed
    for (int r = 0; r < Snap::NROWS; r++) {
      if (!k->has(r) || (r == Snap::R_AUX && !A.aux)) continue;
      CUDA_OK(cudaMemcpyAsync(snap_src(r), k->rows[r], k->bytes(r), cudaMemcpyDeviceToDevice, stream));
    }
    if (A.frames && k->frames && k->frame_list == frame_list) CUDA_OK(cudaMemcpyAsync(A.frames, k->frames, k->frame_bytes(), cudaMemcpyDeviceToDevice, stream));   // frame
    if (A.acc && k->acc && k->frame_list == frame_list) CUDA_OK(cudaMemcpyAsync(A.acc, k->acc, k->acc_bytes(), cudaMemcpyDeviceToDevice, stream));   // and acceleration rows: only between batches with the same frame list, like the aux rows
    return sync();
  }
  // one launch of the restore kernel (reset.cu) from the entries of k into the rows of this batch: environment e, when d_mask[e] is non-zero (null: every
  // environment), takes entry (unsigned)d_entry[e] % k->n (null: e % k->n), by reset_table's rules.  Enqueued only: no synchronisation, copy or allocation
  bool restore_rows(const Snap *k, const unsigned char *dmask, const int *dentry) {
    void *dst[RR_N] = {A.qpos, A.qvel, A.qacc_ws, A.cst, A.xfrc, A.obs, A.dfilt, A.est, A.aux, row(R_APP), A.frames, A.acc};
    const void *src[RR_N];
    for (int r = 0; r < Snap::NROWS; r++) src[r] = k->has(r) ? k->rows[r] : nullptr;
    src[RR_FRAMES] = k->frames; src[RR_ACC] = k->acc;
    ResetArgs R; std::string err;
    if (!reset_table(R, dst, src, (int)sizeof(real), QW, VW, A.nfr, k->frame_list == frame_list, err)) { set_err(err); return false; }
    R.mask = dmask; R.entry = dentry; R.k = k->n; R.n = n;
    CUDA_OK(launch_reset<real>(R, device, stream));
    launches++;
    return true;
  }
  // ---- the reset bank and the device-masked verbs
  bool set_reset_bank(const Snap *k, const int *envs, int nk) override {
    if (nk < 0) { set_err("cassie_batch_set_reset_bank: k must be >= 0"); return false; }
    if (nk == 0 || !k) { CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream)); snap_delete(bank); bank = nullptr; return true; }   // no launch reads the old bank any more
    if (k->esz != (int)sizeof(real) || k->qw != QW || k->vw != VW || k->device != device) { set_err("cassie_batch_set_reset_bank: the snapshot is of another precision, model or device"); return false; }
    if (!envs && nk > k->n) { set_err("cassie_batch_set_reset_bank: k = " + std::to_string(nk) + " exceeds the snapshot's " + std::to_string(k->n) + " environments (envs is NULL)"); return false; }
    if (envs) for (int i = 0; i < nk; i++) if (envs[i] < 0 || envs[i] >= k->n) {
      set_err("cassie_batch_set_reset_bank: envs[" + std::to_string(i) + "] = " + std::to_string(envs[i]) + " is outside the snapshot's " + std::to_string(k->n) + " environments"); return false; }
    CUDA_OK(cudaSetDevice(device));
    Snap *nb = snap_new(device, nk, k->esz, k->qw, k->vw);
    if (!nb) { set_err("cassie_batch_set_reset_bank: out of device memory"); return false; }
    nb->has_est = k->has_est; nb->has_aux = k->has_aux; nb->has_appl = k->has_appl; nb->frame_list = k->frame_list;
    int *d_envs = nullptr; bool ok = true;
    for (int r = 0; r < Snap::NROWS && ok; r++) if (nb->has(r) && !nb->rows[r]) ok = cudaMalloc(&nb->rows[r], nb->bytes(r)) == cudaSuccess;
    if (ok && k->frames) ok = cudaMalloc(&nb->frames, nb->frame_bytes()) == cudaSuccess;
    if (ok && k->acc) ok = cudaMalloc(&nb->acc, nb->acc_bytes()) == cudaSuccess;
    if (ok && envs) ok = cudaMalloc(&d_envs, sizeof(int) * nk) == cudaSuccess && cudaMemcpyAsync(d_envs, envs, sizeof(int) * nk, cudaMemcpyHostToDevice, stream) == cudaSuccess;
    if (ok) {   // the gather runs on the device: entry i of the bank <- environment envs[i] of the snapshot, every row kind the snapshot holds
      void *dst[RR_N]; const void *src[RR_N];
      for (int r = 0; r < Snap::NROWS; r++) { dst[r] = nb->has(r) ? nb->rows[r] : nullptr; src[r] = k->has(r) ? k->rows[r] : nullptr; }
      dst[RR_FRAMES] = nb->frames; src[RR_FRAMES] = k->frames; dst[RR_ACC] = nb->acc; src[RR_ACC] = k->acc;
      ResetArgs R; std::string err;
      if (!reset_table(R, dst, src, k->esz, k->qw, k->vw, (int)(k->frame_list.size() / 2), true, err)) { set_err(err); ok = false; }
      else {
        R.mask = nullptr; R.entry = d_envs; R.k = k->n; R.n = nk;
        const cudaError_t e = launch_reset<real>(R, device, stream);
        if (e != cudaSuccess) { set_err(std::string("cassie_batch_set_reset_bank: ") + cudaGetErrorString(e)); ok = false; }
      }
    } else set_err("cassie_batch_set_reset_bank: out of device memory");
    const cudaError_t es = cudaStreamSynchronize(stream);   // the gather is done (and no launch reads the old bank) before anything is freed
    cudaFree(d_envs);
    if (ok && es != cudaSuccess) { set_err(std::string("cassie_batch_set_reset_bank: ") + cudaGetErrorString(es)); ok = false; }
    if (!ok) { snap_delete(nb); return false; }
    snap_delete(bank); bank = nb;
    return true;
  }
  int reset_bank_size() const override { return bank ? bank->n : 0; }
  // a pointer the device-masked verbs accept: device or managed memory of the batch's device (a host array passed by mistake is refused, not launched)
  bool device_rows(const void *p, const char *verb, const char *what) {
    if (!p) { set_err(std::string(verb) + ": " + what + " is required"); return false; }
    cudaPointerAttributes at{};
    if (cudaPointerGetAttributes(&at, p) != cudaSuccess) { cudaGetLastError(); set_err(std::string(verb) + ": " + what + " is not a CUDA pointer"); return false; }
    if ((at.type != cudaMemoryTypeDevice && at.type != cudaMemoryTypeManaged) || at.device != device) {
      set_err(std::string(verb) + ": " + what + " must be device or managed memory of device " + std::to_string(device) + " (a host array cannot be read by the launch)"); return false; }
    return true;
  }
  bool reset_where(const void *d_mask, const void *d_entry) override {
    const char *verb = "cassie_batch_reset_where";
    if (!bank) { set_err(std::string(verb) + ": no reset bank (cassie_batch_set_reset_bank first)"); return false; }
    if (!device_rows(d_mask, verb, "the mask") || (d_entry && !device_rows(d_entry, verb, "the entry array"))) return false;
    if (est_filter) { set_err(std::string(verb) + ": the host-side estimator filters are on (cassie_batch_enable_estimator_filter): they cannot follow a device reset"); return false; }
    if (legacy) { set_err(std::string(verb) + ": the batch belongs to a cassie_sim_t, whose host mirrors would overwrite the reset"); return false; }
    CUDA_OK(cudaSetDevice(device));
    return restore_rows(bank, (const unsigned char *)d_mask, (const int *)d_entry);
  }
  bool forward_where(const void *d_mask) override {
    const char *verb = "cassie_batch_forward_where";
    if (!device_rows(d_mask, verb, "the mask")) return false;
    if (launch_lends_ext(row_state(), launch_kind(1) == 1)) {   // step_range would lend the chain twin's contact rows here
      set_err(std::string(verb) + ": this batch gets model-valued contact rows at its first extended launch; run cassie_batch_step or cassie_batch_forward once first"); return false; }
    A.mask = (const unsigned char *)d_mask; const bool ok = step(0, 1); A.mask = nullptr;
    return ok;
  }
  bool close_loops(const void *d_mask, int max_iter, double tol) override {
    const std::string verb = "cassie_batch_close_loops";
    if (d_mask && !device_rows(d_mask, verb.c_str(), "the mask")) return false;
    if (max_iter < 1 || max_iter > LOOP_MAX_ITER) { set_err(verb + ": max_iter must be between 1 and " + std::to_string(LOOP_MAX_ITER)); return false; }
    if (!(tol > 0) || !std::isfinite(tol)) { set_err(verb + ": tol must be finite and > 0"); return false; }
    if (legacy) { set_err(verb + ": the batch belongs to a cassie_sim_t, whose host mirrors would overwrite the closed state"); return false; }
    LoopArgs<real> L; std::string err;
    if (!loop_table(hm, L.T, err)) { set_err(verb + ": " + err); return false; }
    CUDA_OK(cudaSetDevice(device));
    if (!d_loops) { CUDA_OK(cudaMalloc(&d_loops, sizeof(real) * n * LOOP_SLOT)); CUDA_OK(cudaMemsetAsync(d_loops, 0, sizeof(real) * n * LOOP_SLOT, stream)); }
    if (L.T.nrow == 0) return true;   // no connect equality: nothing to close
    L.model = d_model; L.qpos = A.qpos; L.qpos_w = QW; L.qvel = A.qvel; L.qvel_w = VW; L.bpos = A.bpos; L.status = d_loops;
    L.mask = (const unsigned char *)d_mask; L.n = n; L.max_iter = max_iter; L.tol = (real)tol;
    CUDA_OK(launch_loops<real>(L, device, stream));
    launches++;
    return true;
  }
  bool get_loop_status(double *residual, int *iterations, double *vel_residual) override {
    if (!d_loops) { set_err("cassie_batch_get_loop_status: no cassie_batch_close_loops call yet"); return false; }
    CUDA_OK(cudaSetDevice(device));
    h_tmp.resize((size_t)n * LOOP_SLOT);
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), d_loops, sizeof(real) * n * LOOP_SLOT, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) {
      const real *r = &h_tmp[(size_t)e * LOOP_SLOT];
      if (residual) residual[e] = (double)r[0];
      if (iterations) iterations[e] = (int)r[1];
      if (vel_residual) vel_residual[e] = (double)r[2];
    }
    return true;
  }
  bool set_ik(const char *const *names, const int *kinds, const int *frames, const double *weights, int count) override {
    const std::string verb = "cassie_batch_set_ik";
    if (count < 0 || count > IK_MAX || (count > 0 && (!names || !kinds || !weights))) { set_err(verb + ": between 0 and " + std::to_string(IK_MAX) + " targets, with names, kinds and weights"); return false; }
    if (legacy) { set_err(verb + ": the batch belongs to a cassie_sim_t, whose host mirrors would overwrite the solved state"); return false; }
    std::vector<int> body(count), frame(count); std::vector<double> pos(3 * count), quat(4 * count), w;
    if (count > 0) w.assign(weights, weights + 6 * count);
    for (int t = 0; t < count; t++) {
      double row[FT_W]; std::string err;
      if (frame_table_row(hm, names[t], kinds[t], row, err) < 0) { set_err(verb + ": " + err); return false; }
      body[t] = (int)row[FT_BODY]; frame[t] = frames ? frames[t] : IK_WORLD;
      if (frame[t] != IK_WORLD && frame[t] != IK_ROOT) { set_err(verb + ": target " + std::to_string(t) + ": frame must be CASSIE_IK_WORLD or CASSIE_IK_ROOT"); return false; }
      for (int c = 0; c < 3; c++) pos[3 * t + c] = row[FT_POS + c];
      for (int c = 0; c < 4; c++) quat[4 * t + c] = row[FT_QUAT + c];
      bool any = false;
      for (int c = 0; c < 6; c++) { const double x = w[6 * t + c]; if (!(x >= 0) || !std::isfinite(x)) { set_err(verb + ": target " + std::to_string(t) + ": weights must be finite and >= 0"); return false; } any |= x > 0; }
      if (!any) { set_err(verb + ": target " + std::to_string(t) + ": every weight is zero"); return false; }
    }
    IkTable<real> I; std::string err;
    if (count > 0 && !ik_table<real>(hm, count, body.data(), frame.data(), pos.data(), quat.data(), w.data(), I, err)) { set_err(verb + ": " + err); return false; }
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaFree(d_ikt)); CUDA_OK(cudaFree(d_ik)); d_ikt = d_ik = nullptr; ik_n = 0;
    if (count > 0) {
      CUDA_OK(cudaMalloc(&d_ikt, sizeof(real) * n * IK_MAX * IK_TW)); CUDA_OK(cudaMemset(d_ikt, 0, sizeof(real) * n * IK_MAX * IK_TW));
      CUDA_OK(cudaMalloc(&d_ik, sizeof(real) * n * IK_SLOT)); CUDA_OK(cudaMemset(d_ik, 0, sizeof(real) * n * IK_SLOT));
      ik_n = count; ik_body = body; ik_frame = frame; ik_pos = pos; ik_quat = quat; ik_w = w;
    }
    return true;
  }
  bool solve_ik(const void *d_mask, int max_iter, double tol, int velocities) override {
    const std::string verb = "cassie_batch_solve_ik";
    if (legacy) { set_err(verb + ": the batch belongs to a cassie_sim_t, whose host mirrors would overwrite the solved state"); return false; }
    if (!ik_n) { set_err(verb + ": no target list (cassie_batch_set_ik)"); return false; }
    if (d_mask && !device_rows(d_mask, verb.c_str(), "the mask")) return false;
    if (max_iter < 1 || max_iter > IK_MAX_ITER) { set_err(verb + ": max_iter must be between 1 and " + std::to_string(IK_MAX_ITER)); return false; }
    if (!(tol > 0) || !std::isfinite(tol)) { set_err(verb + ": tol must be finite and > 0"); return false; }
    if (velocities != 0 && velocities != 1) { set_err(verb + ": velocities must be 0 or 1"); return false; }
    IkArgs<real> K; std::string err;
    if (!ik_table<real>(hm, ik_n, ik_body.data(), ik_frame.data(), ik_pos.data(), ik_quat.data(), ik_w.data(), K.I, err)) { set_err(verb + ": " + err); return false; }
    CUDA_OK(cudaSetDevice(device));
    K.model = d_model; K.qpos = A.qpos; K.qpos_w = QW; K.qvel = A.qvel; K.qvel_w = VW; K.bpos = A.bpos; K.targets = d_ikt; K.status = d_ik;
    K.mask = (const unsigned char *)d_mask; K.n = n; K.max_iter = max_iter; K.velocities = velocities; K.tol = (real)tol;
    K.loop_tol = (real)std::min(tol, sizeof(real) == sizeof(float) ? IK_LOOP_TOL_F : IK_LOOP_TOL_D);
    CUDA_OK(launch_ik<real>(K, device, stream));
    launches++;
    return true;
  }
  bool get_ik_status(double *status) override {
    if (!d_ik) { set_err("cassie_batch_get_ik_status: no target list (cassie_batch_set_ik)"); return false; }
    CUDA_OK(cudaSetDevice(device));
    h_tmp.resize((size_t)n * IK_SLOT);
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), d_ik, sizeof(real) * n * IK_SLOT, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (size_t i = 0; i < (size_t)n * IK_SLOT; i++) status[i] = (double)h_tmp[i];
    return true;
  }
  bool rebuild_model() override {
    CUDA_OK(cudaSetDevice(device));
    DevModel<real> *hmodel = (DevModel<real> *)calloc(1, model_bytes<real>()); std::string err; BuildInfo info;
    if (!build_dev_model(hm, *hmodel, err, &info)) { free(hmodel); set_err(err); return false; }
    if (A.bpos) hmodel->robot_reach = rows_reach(*hmodel);   // per-environment body offsets: the broad phase's bound covers every row
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaMemcpy(d_model, hmodel, model_bytes<real>(), cudaMemcpyHostToDevice));
    h_model_copy = *hmodel; free(hmodel);
    return true;
  }
  bool copy_model_from(BatchBase *other) override {
    Batch<real> *src = dynamic_cast<Batch<real> *>(other);
    if (!src || src->n != n || src->hm.nq != hm.nq || src->hm.nbody != hm.nbody) { set_err("copy: the two simulators differ in model, size or precision"); return false; }
    CUDA_OK(cudaSetDevice(device));
    hm = src->hm;
    if (!rebuild_model()) return false;
    { RowState st = row_state(); RowPlan p; copy_from(st, p, src->row_state());   // what the source lacks is dropped first, top down
      if (!run(p)) return false;
      for (int b = R_CENV; b < R_APP; b++)
        if (src->row(b) ? !copy_rows(b, src) : row(b) && !drop(b)) return false;   // (the constant rows: the others were dropped above)
      lent = st.lent; }
    if (!src->d_terrain && !clear_env_hfield()) return false;
    if (src->d_genv) { if (!ensure_genv()) return false; CUDA_OK(cudaMemcpyAsync(d_genv, src->d_genv, sizeof(real) * n * GEOM_ENV_W, cudaMemcpyDeviceToDevice, stream)); }
    else if (!clear_env_geoms()) return false;
    for (int k = 0; k < MGS; k++) ge_host[k] = src->ge_host[k];
    if (src->d_terrain) {   // the selection row and the height field's mirror (its slots came with the rows above)
      if (!d_terrain) { CUDA_OK(cudaMalloc(&d_terrain, sizeof(int) * n)); A.terrain = d_terrain; }
      CUDA_OK(cudaMemcpyAsync(d_terrain, src->d_terrain, sizeof(int) * n, cudaMemcpyDeviceToDevice, stream));
      hf_host = src->hf_host;
    }
    if (src->d_camenv && src->cam.k == cam.k) {   // the per-environment camera mounts, when the two batches hold as many cameras
      ce_host = src->ce_host;
      CUDA_OK(cudaStreamSynchronize(src->stream)); CUDA_OK(cudaStreamSynchronize(stream));
      const size_t w = (size_t)n * cam.k * CAMENV_SLOT;
      if (!d_camenv) CUDA_OK(cudaMalloc(&d_camenv, sizeof(real) * w));
      CUDA_OK(cudaMemcpy(d_camenv, src->d_camenv, sizeof(real) * w, cudaMemcpyDeviceToDevice));
    } else if (!clear_env_cameras()) return false;
    if (src->A.sn.rows) {   // the sensor models and the generator rows: a copy draws what its source would
      if (!A.sn.rows && !alloc_sensors()) return false;
      CUDA_OK(cudaStreamSynchronize(src->stream)); CUDA_OK(cudaStreamSynchronize(stream));
      CUDA_OK(cudaMemcpy((void *)A.sn.rows, src->A.sn.rows, sizeof(real) * n * SN_W, cudaMemcpyDeviceToDevice));
      CUDA_OK(cudaMemcpy(A.sn.rng, src->A.sn.rng, sizeof(int) * n * SR_W, cudaMemcpyDeviceToDevice));
    } else if (!clear_env_sensors()) return false;
    if (src->d_hfield) {
      const size_t cells = (size_t)hm.hfield_nrow[0] * hm.hfield_ncol[0] * src->A.n_terrain;
      std::vector<float> tmp(cells); CUDA_OK(cudaMemcpy(tmp.data(), src->d_hfield, sizeof(float) * cells, cudaMemcpyDeviceToHost));
      if (!set_hfield(tmp.data(), src->A.n_terrain)) return false;
    }
    return sync();
  }
  // ---- per-environment placement of the static planes / boxes (stairs and slopes that differ between environments)
  bool ensure_genv() {
    if (d_genv) return true;
    CUDA_OK(cudaSetDevice(device));
    std::vector<real> row(GEOM_ENV_W), all((size_t)n * GEOM_ENV_W); init_genv_row(h_model_copy, row.data());
    for (int e = 0; e < n; e++) memcpy(&all[(size_t)e * GEOM_ENV_W], row.data(), sizeof(real) * GEOM_ENV_W);
    CUDA_OK(cudaMalloc(&d_genv, sizeof(real) * n * GEOM_ENV_W));
    CUDA_OK(cudaMemcpyAsync(d_genv, all.data(), sizeof(real) * n * GEOM_ENV_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    A.genv = d_genv;
    return true;
  }
  // slot k of every row <- slots[n][GE_SLOT]: one strided copy, the rest of the rows is not moved
  bool put_genv_slot(int k, const std::vector<real> &slots) {
    CUDA_OK(cudaMemcpy2DAsync(d_genv + GE_SLOT * k, sizeof(real) * GEOM_ENV_W, slots.data(), sizeof(real) * GE_SLOT, sizeof(real) * GE_SLOT, n, cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  std::vector<double> &ge_mirror(int g, int k) {   // the body-frame placement every environment sees; starts as the shared one
    std::vector<double> &h = ge_host[k];
    if (h.empty()) { h.resize((size_t)n * 10);
      for (int e = 0; e < n; e++) { double *r = &h[(size_t)e * 10]; for (int c = 0; c < 3; c++) { r[c] = hm.geom_pos[3 * g + c]; r[7 + c] = hm.geom_size[3 * g + c]; } for (int c = 0; c < 4; c++) r[3 + c] = hm.geom_quat[4 * g + c]; } }
    return h;
  }
  bool set_env_geom(int g, const double *pos, const double *quat, const double *size, const unsigned char *mask) override {
    std::string err; const int k = env_geom_check(hm, geom_dev, g, err);
    if (k < 0) { set_err("cassie_batch_set_env_geom_pose: " + err); return false; }
    if (!ensure_genv()) return false;
    // the selected environments' slots from their new placement; the others keep the slot they have (read back: 64 B per environment)
    std::vector<real> slots((size_t)n * GE_SLOT);
    CUDA_OK(cudaMemcpy2DAsync(slots.data(), sizeof(real) * GE_SLOT, d_genv + GE_SLOT * k, sizeof(real) * GEOM_ENV_W, sizeof(real) * GE_SLOT, n, cudaMemcpyDeviceToHost, stream));
    CUDA_OK(cudaStreamSynchronize(stream));
    std::vector<double> &h = ge_mirror(g, k);
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      double *r = &h[(size_t)e * 10];
      if (pos) for (int c = 0; c < 3; c++) r[c] = pos[(size_t)e * 3 + c];
      if (quat) for (int c = 0; c < 4; c++) r[3 + c] = quat[(size_t)e * 4 + c];
      if (size) for (int c = 0; c < 3; c++) r[7 + c] = size[(size_t)e * 3 + c];
      env_geom_slot(hm, g, r, r + 3, r + 7, &slots[(size_t)e * GE_SLOT]);
    }
    return put_genv_slot(k, slots);
  }
  bool get_env_geom(int g, double *pos, double *quat, double *size) override {
    std::string err; const int k = env_geom_check(hm, geom_dev, g, err);
    if (k < 0) { set_err("cassie_batch_get_env_geom_pose: " + err); return false; }
    for (int e = 0; e < n; e++) {
      const double *r = ge_host[k].empty() ? nullptr : &ge_host[k][(size_t)e * 10];
      for (int c = 0; c < 3; c++) { if (pos) pos[(size_t)e * 3 + c] = r ? r[c] : hm.geom_pos[3 * g + c]; if (size) size[(size_t)e * 3 + c] = r ? r[7 + c] : hm.geom_size[3 * g + c]; }
      if (quat) for (int c = 0; c < 4; c++) quat[(size_t)e * 4 + c] = r ? r[3 + c] : hm.geom_quat[4 * g + c];
    }
    return true;
  }
  bool clear_env_geoms() override {   // the height field's position and size go back to the shared ones too; a terrain selection stays
    for (int k = 0; k < MGS; k++) ge_host[k].clear();
    hf_host.clear();
    if (!d_genv) return true;
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaFree(d_genv)); d_genv = nullptr; A.genv = nullptr;
    return !d_terrain || (ensure_genv() && put_hf_slots());   // the F_TR instances read the height field's slot: fresh rows with the shared one
  }
  bool shared_geom_changed(int g) override {
    const int k = g >= 0 && g < hm.ngeom ? geom_dev[g] - MG : -1;
    if (k < 0 || k >= MGS) return true;
    ge_host[k].clear();
    if (g == hfield_geom(hm)) { hf_host.clear(); if (d_terrain) return put_hf_slots(); }
    if (!d_genv) return true;
    std::vector<real> row(GEOM_ENV_W), slots((size_t)n * GE_SLOT); init_genv_row(h_model_copy, row.data());
    for (int e = 0; e < n; e++) memcpy(&slots[(size_t)e * GE_SLOT], &row[GE_SLOT * k], sizeof(real) * GE_SLOT);
    return put_genv_slot(k, slots);
  }
  // ---- per-environment terrain (terrain curricula): which bank entry each environment stands on, and where and how large its height field is
  int hf_slot(const char *verb) {   // the height field's static slot, or -1 with an error
    const int g = hfield_geom(hm), k = g >= 0 ? geom_dev[g] - MG : -1;
    if (hm.nhfield != 1 || k < 0 || k >= MGS) { set_err(std::string(verb) + ": this model has no height field"); return -1; }
    return k;
  }
  void hf_shared(double *r) { const int g = hfield_geom(hm); for (int c = 0; c < 3; c++) r[c] = hm.geom_pos[3 * g + c]; for (int c = 0; c < 4; c++) r[3 + c] = hm.hfield_size[c]; }
  bool put_hf_slots() {   // the height field's slot of every row from the mirror (or the shared position and size)
    const int g = hfield_geom(hm), k = geom_dev[g] - MG;
    std::vector<real> slots((size_t)n * GE_SLOT); double sh[7]; hf_shared(sh);
    for (int e = 0; e < n; e++) { const double *r = hf_host.empty() ? sh : &hf_host[(size_t)e * 7]; env_hfield_slot(hm, g, r, r + 3, &slots[(size_t)e * GE_SLOT]); }
    return put_genv_slot(k, slots);
  }
  bool set_env_hfield(const int *terrain, const double *pos, const double *size, const unsigned char *mask) override {
    const char *verb = "cassie_batch_set_env_hfield";
    if (hf_slot(verb) < 0) return false;
    for (int e = 0; e < n; e++) {   // every masked environment is checked before anything changes
      if (mask && !mask[e]) continue;
      const std::string at = std::string(verb) + ": environment " + std::to_string(e) + ": ";
      if (terrain && (terrain[e] < 0 || terrain[e] >= A.n_terrain)) { set_err(at + "terrain " + std::to_string(terrain[e]) + " is outside [0, " + std::to_string(A.n_terrain) + ")"); return false; }
      if (pos && !std::isfinite(pos[3 * e] + pos[3 * e + 1] + pos[3 * e + 2])) { set_err(at + "pos is not finite"); return false; }
      if (size) { const std::string w = hfield_size_check(size + 4 * (size_t)e); if (!w.empty()) { set_err(at + w); return false; } }
    }
    CUDA_OK(cudaSetDevice(device));
    if (!ensure_genv()) return false;
    std::vector<int> t(n);
    if (d_terrain) { CUDA_OK(cudaMemcpyAsync(t.data(), d_terrain, sizeof(int) * n, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream)); }   // it may have been written on the device
    else for (int e = 0; e < n; e++) t[e] = e % A.n_terrain;
    if (hf_host.empty()) { double sh[7]; hf_shared(sh); hf_host.resize((size_t)n * 7); for (int e = 0; e < n; e++) memcpy(&hf_host[(size_t)e * 7], sh, sizeof sh); }
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      if (terrain) t[e] = terrain[e];
      if (pos) for (int c = 0; c < 3; c++) hf_host[(size_t)e * 7 + c] = pos[3 * (size_t)e + c];
      if (size) for (int c = 0; c < 4; c++) hf_host[(size_t)e * 7 + 3 + c] = size[4 * (size_t)e + c];
    }
    if (!d_terrain) CUDA_OK(cudaMalloc(&d_terrain, sizeof(int) * n));
    CUDA_OK(cudaMemcpyAsync(d_terrain, t.data(), sizeof(int) * n, cudaMemcpyHostToDevice, stream));
    A.terrain = d_terrain;
    return put_hf_slots();
  }
  bool get_env_hfield(int *terrain, double *pos, double *size) override {
    if (hf_slot("cassie_batch_get_env_hfield") < 0) return false;
    CUDA_OK(cudaSetDevice(device));
    if (terrain) {
      if (d_terrain) { CUDA_OK(cudaMemcpyAsync(terrain, d_terrain, sizeof(int) * n, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream)); }
      else for (int e = 0; e < n; e++) terrain[e] = e % A.n_terrain;
    }
    double sh[7]; hf_shared(sh);
    for (int e = 0; e < n; e++) {
      const double *r = hf_host.empty() ? sh : &hf_host[(size_t)e * 7];
      if (pos) for (int c = 0; c < 3; c++) pos[3 * (size_t)e + c] = r[c];
      if (size) for (int c = 0; c < 4; c++) size[4 * (size_t)e + c] = r[3 + c];
    }
    return true;
  }
  bool clear_env_hfield() override {   // back to terrain e % K and the shared placement and size: the slot as the model block has it
    hf_host.clear();
    if (d_terrain) { CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(d_terrain)); d_terrain = nullptr; A.terrain = nullptr; }
    const int g = hfield_geom(hm);
    return g < 0 || !d_genv || shared_geom_changed(g);
  }
  bool set_hfield_size(const double *size) override {
    const char *verb = "cassie_batch_set_hfield_size";
    if (hf_slot(verb) < 0) return false;
    if (!size) { set_err(std::string(verb) + ": size is required"); return false; }
    const std::string w = hfield_size_check(size);
    if (!w.empty()) { set_err(std::string(verb) + ": " + w); return false; }
    const int g = hfield_geom(hm);
    for (int c = 0; c < 4; c++) hm.hfield_size[c] = size[c];
    const double z = std::max(size[2], size[3]);
    hm.geom_rbound[g] = std::sqrt(size[0] * size[0] + size[1] * size[1] + z * z);   // the model compiler's bound for the new size
    return rebuild_model() && shared_geom_changed(g);   // every environment's height-field position and size follow the shared ones
  }
  // ---- per-environment body offsets (loads, trays, link offsets): MuJoCo's body_pos per environment, read by the F_BP instances' kinematics and by the
  // ray and camera kernels
  real rows_reach(const DevModel<real> &d) const {   // the block's robot_reach for the rows: build_dev_model's bound, the largest over the environments
    const int nb3 = 3 * hm.nbody; double r = 0;
    for (int e = 0; e < n; e++) r = std::max(r, robot_reach_of(hm, &bp_host[(size_t)e * nb3], d.root_body, d.xb, geom_dev));
    return (real)(r * 1.05 + 0.05);
  }
  bool put_bpos() {   // the device rows and the block's robot_reach from the mirror
    const int nb3 = 3 * hm.nbody;
    std::vector<real> all((size_t)n * BP_W, real(0));
    for (int e = 0; e < n; e++) for (int i = 0; i < nb3; i++) all[(size_t)e * BP_W + i] = (real)bp_host[(size_t)e * nb3 + i];
    return push(R_BPOS, all);
  }
  bool put_reach() {   // after the offset rows changed (a launch in flight reads the block: the caller synchronised)
    h_model_copy.robot_reach = rows_reach(h_model_copy);
    CUDA_OK(cudaMemcpy(&d_model->robot_reach, &h_model_copy.robot_reach, sizeof(real), cudaMemcpyHostToDevice));
    return true;
  }
  bool set_env_body_pos(const double *pos, const unsigned char *mask) override {
    const std::string verb = "cassie_batch_set_env_body_pos";
    if (!pos) { set_err(verb + ": pos is required"); return false; }
    const int nb = hm.nbody, nb3 = 3 * nb;
    for (int e = 0; e < n; e++) {   // every masked environment is checked before anything changes
      if (mask && !mask[e]) continue;
      const double *now = bp_host.empty() ? hm.body_pos.data() : &bp_host[(size_t)e * nb3];
      for (int b = 0; b < nb; b++) {
        const double *p = pos + (size_t)e * nb3 + 3 * b;
        const std::string at = verb + ": environment " + std::to_string(e) + ", body " + hm.names_body[b] + ": ";
        if (!std::isfinite(p[0]) || !std::isfinite(p[1]) || !std::isfinite(p[2])) { set_err(at + "pos is not finite"); return false; }
        if (p[0] == now[3 * b] && p[1] == now[3 * b + 1] && p[2] == now[3 * b + 2]) continue;
        const std::string w = env_body_pos_check(hm, b, h_model_copy.xb);
        if (!w.empty()) { set_err(at + "the offset of " + w + " cannot change"); return false; }
      }
    }
    if (!rows_rule(own, R_BPOS)) return false;
    if (bp_host.empty()) { bp_host.resize((size_t)n * nb3); for (int e = 0; e < n; e++) memcpy(&bp_host[(size_t)e * nb3], hm.body_pos.data(), sizeof(double) * nb3); }
    for (int e = 0; e < n; e++) if (!mask || mask[e]) memcpy(&bp_host[(size_t)e * nb3], pos + (size_t)e * nb3, sizeof(double) * nb3);
    return put_bpos();
  }
  bool get_env_body_pos(double *pos) override {
    if (!pos) { set_err("cassie_batch_get_env_body_pos: pos is required"); return false; }
    const int nb3 = 3 * hm.nbody;
    for (int e = 0; e < n; e++) memcpy(pos + (size_t)e * nb3, bp_host.empty() ? hm.body_pos.data() : &bp_host[(size_t)e * nb3], sizeof(double) * nb3);
    return true;
  }
  bool clear_env_body_pos() override { return rows_rule(release, R_BPOS); }   // back to the model's offsets and the instances that ran before
  void model_bpos_rows() {   // the mirror of offset rows holding the model's offsets in every environment
    const int nb3 = 3 * hm.nbody;
    bp_host.resize((size_t)n * nb3); for (int e = 0; e < n; e++) memcpy(&bp_host[(size_t)e * nb3], hm.body_pos.data(), sizeof(double) * nb3);
  }
  // ---- per-environment actuators (actuator latency and torque saturation: sim-to-real randomisation): ctrlrange, no-load speed and torque delay per
  // motor, read by the F_AC instances' motor stage and actuation.  The device rows are what the environments run with: a caller may have written them
  // through the "actuators" device pointer.  The mirror keeps the doubles the verb was last given, so that get reports them exactly (rpm included)
  // wherever the device still holds what they stored.
  static real act_row_value(const double *a, int f) { return f == 2 ? (real)(a[2] * 2 * M_PI / 60) : (real)a[f]; }   // wmax: build_dev_model's expression
  static int act_delay_host(real v) { return (int)(v > real(0) ? (v < real(AC_MAXDELAY) ? v : real(AC_MAXDELAY)) : real(0)); }   // the kernel's act_delay_index
  static constexpr int AC_FIELD[4] = {AC_LO, AC_HI, AC_WMAX, AC_DELAY};
  void model_act(int i, double *a) const {   // motor i as the model has it: lo, hi (the clamp the block holds), rpm, the reference's delay
    a[0] = (double)h_model_copy.act_ctrl_lo[i]; a[1] = (double)h_model_copy.act_ctrl_hi[i]; a[2] = hm.actuator_user[i]; a[3] = AC_MAXDELAY;
  }
  void model_act_rows(std::vector<real> &all) {   // the mirror and the rows holding the model's actuators in every environment
    const int nu = hm.nu;
    ac_host.resize((size_t)n * nu * 4); all.assign((size_t)n * ACT_W, real(0));
    for (int e = 0; e < n; e++) for (int i = 0; i < nu; i++) {
      double *a = &ac_host[((size_t)e * nu + i) * 4]; model_act(i, a);
      for (int f = 0; f < 4; f++) all[(size_t)e * ACT_W + AC_FIELD[f] + i] = act_row_value(a, f);
    }
  }
  bool set_env_actuators(const double *ctrlrange, const double *rpm, const int *delay, const unsigned char *mask) override {
    const std::string verb = "cassie_batch_set_env_actuators";
    const int nu = hm.nu;
    if (nu > MU) { set_err(verb + ": the model has more than " + std::to_string(MU) + " actuators"); return false; }
    const std::string why = env_actuators_check(n, nu, ctrlrange, rpm, delay, mask);   // every masked value is checked before anything changes
    if (!why.empty()) { set_err(verb + ": " + why); return false; }
    if (!rows_rule(own, R_ACT)) return false;
    std::vector<real> all;
    if (!A.act) model_act_rows(all);   // the first call: every environment starts from the model's actuators
    else if (!pull(R_ACT, all)) return false;   // unmasked environments keep what their rows hold, also when it was written on the device
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      for (int i = 0; i < nu; i++) {
        const size_t k = (size_t)e * nu + i; double *a = &ac_host[k * 4]; real *r = &all[(size_t)e * ACT_W];
        if (ctrlrange) { a[0] = ctrlrange[2 * k]; a[1] = ctrlrange[2 * k + 1]; r[AC_LO + i] = act_row_value(a, 0); r[AC_HI + i] = act_row_value(a, 1); }
        if (rpm) { a[2] = rpm[k]; r[AC_WMAX + i] = act_row_value(a, 2); }
        if (delay) { a[3] = delay[k]; r[AC_DELAY + i] = act_row_value(a, 3); }
      }
    }
    return push(R_ACT, all);
  }
  // what every environment runs with: a value the device row still holds as the verb stored it is reported as the verb was given it; one written on the
  // device is reported from the row (rpm = wmax * 60 / 2 pi, the delay as the kernel reads it)
  bool get_env_actuators(double *ctrlrange, double *rpm, int *delay) override {
    const int nu = hm.nu;
    std::vector<real> all;
    if (!pull(R_ACT, all)) return false;
    for (int e = 0; e < n; e++) for (int i = 0; i < nu; i++) {
      const size_t k = (size_t)e * nu + i;
      double m[4]; model_act(i, m);
      double v[4] = {m[0], m[1], m[2], m[3]};
      if (A.act) {
        const double *a = &ac_host[k * 4];
        for (int f = 0; f < 4; f++) {
          const real dv = all[(size_t)e * ACT_W + AC_FIELD[f] + i];
          if (dv == act_row_value(a, f)) v[f] = a[f];
          else v[f] = f == 2 ? (double)dv * 60 / (2 * M_PI) : (f == 3 ? (double)act_delay_host(dv) : (double)dv);
        }
      }
      if (ctrlrange) { ctrlrange[2 * k] = v[0]; ctrlrange[2 * k + 1] = v[1]; }
      if (rpm) rpm[k] = v[2];
      if (delay) delay[k] = (int)v[3];
    }
    return true;
  }
  bool clear_env_actuators() override { return rows_rule(release, R_ACT); }   // back to the model's actuators and the instances that ran before
  // ---- per-environment mechanics (link inertia, rotor armature, leaf springs: sim-to-real randomisation): MuJoCo's body_inertia, dof_armature and the
  // jnt_stiffness / qpos_spring of the hinges per environment, read by the F_MC instances' cinert, CRB and passive phases.  As with the actuator rows,
  // the device rows are what the environments run with, and the mirror keeps the doubles the verb was last given.
  int mech_host_w() const { return 3 * hm.nbody + hm.nv + 2 * hm.njnt; }   // the mirror per environment: inertia [nbody][3], armature [nv], stiffness [njnt], springref [njnt]
  int mech_slot(int k) const {   // the row slot of mirror entry k, or -1 where the kernel reads the block (the extra free body's dofs, non-hinge springs)
    const int nb3 = 3 * hm.nbody, nv = hm.nv, nj = hm.njnt;
    if (k < nb3) return MC_INERTIA + k;
    if ((k -= nb3) < nv) return k < h_model_copy.nv ? MC_ARMATURE + k : -1;
    const int base = (k -= nv) < nj ? MC_STIFF : MC_SPRING, j = k % nj;
    return hm.jnt_type[j] == JNT_HINGE ? base + hm.jnt_dofadr[j] : -1;
  }
  double block_mech(int k) const {   // mirror entry k as the shared block has it (what get reports where the kernel reads the block)
    const int nb3 = 3 * hm.nbody, nv = hm.nv, nj = hm.njnt;
    if (k < nb3) return hm.body_inertia[k];
    if ((k -= nb3) < nv) return hm.dof_armature[k];
    return (k -= nv) < nj ? hm.jnt_stiffness[k] : hm.qpos_spring[hm.jnt_qposadr[k - nj]];
  }
  void model_mech_rows(std::vector<real> &all) {   // the mirror and the rows holding the model's values in every environment (a non-hinge dof's slots too, though the kernel reads the block there)
    const int w = mech_host_w();
    mc_host.resize((size_t)n * w); all.assign((size_t)n * MECH_W, real(0));
    for (int e = 0; e < n; e++) {
      real *r = &all[(size_t)e * MECH_W];
      for (int k = 0; k < w; k++) { mc_host[(size_t)e * w + k] = block_mech(k); const int sl = mech_slot(k); if (sl >= 0) r[sl] = (real)block_mech(k); }
      for (int i = 0; i < h_model_copy.nv; i++) { const int j = hm.dof_jntid[i]; r[MC_STIFF + i] = (real)hm.jnt_stiffness[j]; r[MC_SPRING + i] = (real)hm.qpos_spring[hm.jnt_qposadr[j]]; }
    }
  }
  bool set_env_mechanics(const double *inertia, const double *armature, const double *stiffness, const double *springref, const unsigned char *mask) override {
    const std::string verb = "cassie_batch_set_env_mechanics";
    const std::string why = env_mechanics_check(hm, n, h_model_copy.xb, h_model_copy.nv, inertia, armature, stiffness, springref, mask);   // every masked value first
    if (!why.empty()) { set_err(verb + ": " + why); return false; }
    if (!rows_rule(own, R_MECH)) return false;
    const int w = mech_host_w(), nb3 = 3 * hm.nbody, nv = hm.nv, nj = hm.njnt;
    std::vector<real> all;
    if (!A.mech) model_mech_rows(all);   // the first call: every environment starts from the model's values
    else if (!pull(R_MECH, all)) return false;   // unmasked environments keep what their rows hold, also when it was written on the device
    const double *part[4] = {inertia, armature, stiffness, springref};
    const int off[5] = {0, nb3, nb3 + nv, nb3 + nv + nj, w};
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      for (int p = 0; p < 4; p++) {
        if (!part[p]) continue;
        const int cnt = off[p + 1] - off[p];
        for (int i = 0; i < cnt; i++) {
          const double v = part[p][(size_t)e * cnt + i]; const int k = off[p] + i, sl = mech_slot(k);
          mc_host[(size_t)e * w + k] = v;
          if (sl >= 0) all[(size_t)e * MECH_W + sl] = (real)v;
        }
      }
    }
    return push(R_MECH, all);
  }
  // what every environment runs with: a value the device row still holds as the verb stored it is reported as the verb was given it, one written on the
  // device from the row; where the kernel reads the block (the extra free body's armature, non-hinge springs), the block's current value
  bool get_env_mechanics(double *inertia, double *armature, double *stiffness, double *springref) override {
    const int w = mech_host_w(), nb3 = 3 * hm.nbody, nv = hm.nv, nj = hm.njnt;
    std::vector<real> all;
    if (!pull(R_MECH, all)) return false;
    double *part[4] = {inertia, armature, stiffness, springref};
    const int off[5] = {0, nb3, nb3 + nv, nb3 + nv + nj, w};
    for (int e = 0; e < n; e++) for (int p = 0; p < 4; p++) {
      if (!part[p]) continue;
      const int cnt = off[p + 1] - off[p];
      for (int i = 0; i < cnt; i++) {
        const int k = off[p] + i, sl = mech_slot(k);
        double v = block_mech(k);
        if (A.mech && sl >= 0) { const real dv = all[(size_t)e * MECH_W + sl]; const double a = mc_host[(size_t)e * w + k]; v = dv == (real)a ? a : (double)dv; }
        part[p][(size_t)e * cnt + i] = v;
      }
    }
    return true;
  }
  bool clear_env_mechanics() override { return rows_rule(release, R_MECH); }   // back to the model's values and the instances that ran before
  // ---- per-environment contact softness (ground stiffness, damping and impedance: sim-to-real randomisation): MuJoCo's geom_solref, geom_solimp and
  // geom_solmix per collision geom and environment, mixed per contact row by the F_CT instances' constraint stage.  The device rows are what the
  // environments run with, and the mirror keeps the doubles the verb was last given.
  int ct_slot(int g) const { return g < 256 && geom_dev[g] >= 0 && geom_dev[g] < MGT ? geom_dev[g] : -1; }   // the device geom of host geom g, or -1: no contact
  static int ct_field(int f) { return f < 2 ? CT_SOLREF + f : (f < 7 ? CT_SOLIMP + f - 2 : CT_SOLMIX); }   // mirror field f (solref 2, solimp 5, solmix 1) -> slot offset
  double model_ct(int g, int f) const { return f < 2 ? hm.geom_solref[2 * g + f] : (f < 7 ? hm.geom_solimp[5 * g + f - 2] : hm.geom_solmix[g]); }
  void model_ct_rows(std::vector<real> &all) {   // the mirror and the rows holding the model's values in every environment
    const int ng = hm.ngeom;
    ct_host.resize((size_t)n * ng * CT_SLOT); all.assign((size_t)n * CONTACT_W, real(0));
    for (int e = 0; e < n; e++) for (int g = 0; g < ng; g++) {
      const int s = ct_slot(g);
      for (int f = 0; f < CT_SLOT; f++) {
        ct_host[((size_t)e * ng + g) * CT_SLOT + f] = model_ct(g, f);
        if (s >= 0) all[(size_t)e * CONTACT_W + CT_SLOT * s + ct_field(f)] = (real)model_ct(g, f);
      }
    }
  }
  bool set_env_contact(const double *solref, const double *solimp, const double *solmix, const unsigned char *mask) override {
    const std::string verb = "cassie_batch_set_env_contact";
    const std::string why = env_contact_check(hm, n, geom_dev, solref, solimp, solmix, mask);   // every masked value first
    if (!why.empty()) { set_err(verb + ": " + why); return false; }
    if (!rows_rule(own, R_CT)) return false;
    const int ng = hm.ngeom;
    std::vector<real> all;
    if (!A.contact) model_ct_rows(all);   // the first call: every environment starts from the model's values
    else if (!pull(R_CT, all)) return false;   // unmasked environments keep what their rows hold, also when it was written on the device
    const double *part[3] = {solref, solimp, solmix};
    const int off[4] = {0, 2, 7, 8};
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      for (int g = 0; g < ng; g++) {
        const int s = ct_slot(g); if (s < 0) continue;   // no collision slot: never in contact, the entry is ignored
        for (int p = 0; p < 3; p++) {
          if (!part[p]) continue;
          const int cnt = off[p + 1] - off[p];
          for (int i = 0; i < cnt; i++) {
            const double v = part[p][((size_t)e * ng + g) * cnt + i]; const int f = off[p] + i;
            ct_host[((size_t)e * ng + g) * CT_SLOT + f] = v;
            all[(size_t)e * CONTACT_W + CT_SLOT * s + ct_field(f)] = (real)v;
          }
        }
      }
    }
    return push(R_CT, all);
  }
  // what every environment runs with: a value the device row still holds as the verb stored it is reported as the verb was given it, one written on the
  // device from the row; geoms without a collision slot report the model's values
  bool get_env_contact(double *solref, double *solimp, double *solmix) override {
    const int ng = hm.ngeom;
    std::vector<real> all;
    if (!pull(R_CT, all)) return false;
    double *part[3] = {solref, solimp, solmix};
    const int off[4] = {0, 2, 7, 8};
    for (int e = 0; e < n; e++) for (int g = 0; g < ng; g++) {
      const int s = ct_slot(g);
      for (int p = 0; p < 3; p++) {
        if (!part[p]) continue;
        const int cnt = off[p + 1] - off[p];
        for (int i = 0; i < cnt; i++) {
          const int f = off[p] + i;
          double v = model_ct(g, f);
          if (A.contact && s >= 0) { const real dv = all[(size_t)e * CONTACT_W + CT_SLOT * s + ct_field(f)]; const double a = ct_host[((size_t)e * ng + g) * CT_SLOT + f]; v = dv == (real)a ? a : (double)dv; }
          part[p][((size_t)e * ng + g) * cnt + i] = v;
        }
      }
    }
    return true;
  }
  bool clear_env_contact() override { return rows_rule(release, R_CT); }   // back to the model's values and the instances that ran before
  // ---- per-environment applied forces (pushes on any body, joint-space disturbances): MuJoCo's xfrc_applied and qfrc_applied per environment.  They are
  // state, as in mjData: reset zeroes them, snapshots carry them.  The device rows are what the environments run with (a write through the device
  // pointer takes effect at the next launch), so the verbs read them back and keep no mirror.  A batch with rows runs f0404 / f2404 where f04 / f24
  // would run, else the chain twins.
  int ap_col(int i) const { const int nvm = h_model_copy.nv; return i < nvm ? i : 32 + (i - nvm); }   // host dof i -> its column in AP_QFRC
  bool enable_applied_forces(bool on) override {
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a launch in flight reads the rows
    if (on) return rows_rule(own, R_APP) && (A.applied || put_model(R_APP));   // the first call: zeroed rows
    if (A.applied && !drop(R_APP)) return false;
    return rows_rule(dropped, R_APP);   // back to the instances that ran before
  }
  bool set_applied_forces(const double *xfrc, const double *qfrc, const unsigned char *mask) override {
    const int nb = hm.nbody, nv = hm.nv;
    for (int e = 0; e < n; e++) {   // every masked value first
      if (mask && !mask[e]) continue;
      for (int b = 0; xfrc && b < nb; b++) for (int k = 0; k < 6; k++) if (!std::isfinite(xfrc[((size_t)e * nb + b) * 6 + k])) {
        const std::string name = (size_t)b < hm.names_body.size() && !hm.names_body[b].empty() ? hm.names_body[b] : std::to_string(b);
        set_err("cassie_batch_set_applied_forces: environment " + std::to_string(e) + ", body " + name + ": xfrc_applied[" + std::to_string(k) + "] is not finite"); return false; }
      for (int i = 0; qfrc && i < nv; i++) if (!std::isfinite(qfrc[(size_t)e * nv + i])) {
        set_err("cassie_batch_set_applied_forces: environment " + std::to_string(e) + ", dof " + std::to_string(i) + ": qfrc_applied is not finite"); return false; }
    }
    std::vector<real> all;
    if (!enable_applied_forces(true) || !pull(R_APP, all)) return false;   // unmasked environments keep what their rows hold
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      real *r = &all[(size_t)e * APPLIED_W];
      if (xfrc) for (int b = 0; b < nb; b++) for (int k = 0; k < 6; k++) r[AP_XFRC + 6 * b + k] = (real)xfrc[((size_t)e * nb + b) * 6 + k];
      if (qfrc) for (int i = 0; i < nv; i++) r[AP_QFRC + ap_col(i)] = (real)qfrc[(size_t)e * nv + i];
    }
    return push(R_APP, all);
  }
  bool get_applied_forces(double *xfrc, double *qfrc) override {   // what the rows hold; zeros without rows
    const int nb = hm.nbody, nv = hm.nv;
    std::vector<real> all;
    if (!pull(R_APP, all)) return false;
    for (int e = 0; e < n; e++) {
      const real *r = &all[(size_t)e * APPLIED_W];
      if (xfrc) for (int b = 0; b < nb; b++) for (int k = 0; k < 6; k++) xfrc[((size_t)e * nb + b) * 6 + k] = (double)r[AP_XFRC + 6 * b + k];
      if (qfrc) for (int i = 0; i < nv; i++) qfrc[(size_t)e * nv + i] = (double)r[AP_QFRC + ap_col(i)];
    }
    return true;
  }
  bool clear_applied_xfrc() override {   // cassie_batch_clear_forces: MuJoCo's xfrc_applied of every environment; qfrc_applied stays (src/cassiemujoco.c:1969-1972)
    if (!A.applied) return true;
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemset2DAsync(row(R_APP) + AP_XFRC, sizeof(real) * APPLIED_W, 0, sizeof(real) * AP_QFRC, n, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  // ---- per-tick trace: the rows are an output, written by step launches only.  The trace instances are twins of the extended chain twins: the rows they
  // need are lent here (env_rows.h), so that a step allocates nothing
  bool set_trace(const int *source, const int *column, int k, int max_ticks) override {
    const std::string verb = "cassie_batch_set_trace: ";
    if (legacy) { set_err(verb + "the batch belongs to a cassie_sim_t"); return false; }
    if (k > 0 && A.cl.rows) { set_err(verb + "the batch has contact lists (cassie_batch_enable_contacts); a trace and contact lists do not combine"); return false; }
    if (k > 0 && A.sn.rows) { set_err(verb + "the batch has sensor models (cassie_batch_set_env_sensors); a trace and sensor models do not combine"); return false; }
    if (k < 0 || k > TRACE_MAX) { set_err(verb + "between 0 and " + std::to_string(TRACE_MAX) + " columns"); return false; }
    std::vector<int> codes((size_t)k);
    int need = 0;
    if (k > 0) {
      if (!source || !column) { set_err(verb + "source and column are required"); return false; }
      if (max_ticks < 1) { set_err(verb + "max_ticks must be at least 1"); return false; }
      static const char *const names[TC_NSRC] = {"qpos", "qvel", "observation", "derived-quantity", "frame"};
      for (int c = 0; c < k; c++) {
        const int src = source[c], col = column[c];
        if (src < 0 || src >= TC_NSRC) { set_err(verb + "column " + std::to_string(c) + ": unknown source " + std::to_string(src)); return false; }
        if (src == TC_AUX && !A.aux) { set_err(verb + "column " + std::to_string(c) + ": derived-quantity columns need cassie_batch_enable_aux"); return false; }
        if (src == TC_FRAME && !A.frames) { set_err(verb + "column " + std::to_string(c) + ": frame columns need cassie_batch_set_frames"); return false; }
        const int width = src == TC_QPOS ? hm.nq : src == TC_QVEL ? hm.nv : src == TC_OBS ? OBS_W : src == TC_AUX ? AUX_W : A.nfr * FRAME_W;
        if (col < 0 || col >= width) { set_err(verb + "column " + std::to_string(c) + ": " + names[src] + " column " + std::to_string(col) + " is outside 0.." + std::to_string(width - 1)); return false; }
        codes[c] = (src << TC_SHIFT) | col;
        if (src >= TC_OBS) need |= 1 << src;
      }
    }
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a launch in flight writes the rows
    CUDA_OK(cudaFree(A.trace.rows)); CUDA_OK(cudaFree((void *)A.trace.cols)); A.trace = TraceArgs<real>{}; tc_ticks = 0;
    if (k == 0) return rows_rule(dropped, R_TRACE);   // back to the instances that ran before
    if (!rows_rule(own, R_TRACE)) return false;
    int *cols = nullptr;
    CUDA_OK(cudaMalloc(&cols, sizeof(int) * k)); CUDA_OK(cudaMemcpy(cols, codes.data(), sizeof(int) * k, cudaMemcpyHostToDevice));
    CUDA_OK(cudaMalloc(&A.trace.rows, sizeof(real) * n * max_ticks * k)); CUDA_OK(cudaMemset(A.trace.rows, 0, sizeof(real) * n * max_ticks * k));
    A.trace.cols = cols; A.trace.k = k; A.trace.T = max_ticks; A.trace.need = need;
    return true;
  }
  bool get_trace(double *out) override {
    if (!A.trace.rows) { set_err("cassie_batch_get_trace: no trace is set (cassie_batch_set_trace)"); return false; }
    if (!out) { set_err("cassie_batch_get_trace: out is required"); return false; }
    return d2h(A.trace.rows, A.trace.T * A.trace.k, A.trace.T * A.trace.k, 0, out);
  }
  int trace_ticks() const override { return tc_ticks; }
  // ---- contact lists: the rows are an output, written by step and forward launches only.  The contact-list instances are twins of the F_FR chain
  // twins: the rows they need are lent as with a trace
  bool enable_contacts(bool on) override {
    if (on && A.trace.rows) { set_err("cassie_batch_enable_contacts: the batch has a per-tick trace (cassie_batch_set_trace); a trace and contact lists do not combine"); return false; }
    if (on && A.sn.rows) { set_err("cassie_batch_enable_contacts: the batch has sensor models (cassie_batch_set_env_sensors); contact lists and sensor models do not combine"); return false; }
    CUDA_OK(cudaSetDevice(device));
    if (on && !A.cl.rows) {
      if (!rows_rule(own, R_CL) || !geom_table()) return false;
      real *rows = nullptr;
      CUDA_OK(cudaMalloc(&rows, sizeof(real) * n * CON_W)); CUDA_OK(cudaMemset(rows, 0, sizeof(real) * n * CON_W));
      A.cl.rows = rows; A.cl.geom = d_gtab;
    }
    if (!on && A.cl.rows) {
      CUDA_OK(cudaStreamSynchronize(stream));   // a launch in flight writes the rows
      CUDA_OK(cudaFree(A.cl.rows)); A.cl = ContactListArgs<real>{};   // (the geom table stays with the batch)
      return rows_rule(dropped, R_CL);   // back to the instances that ran before
    }
    return true;
  }
  // ---- sensor models: a model input like the actuator rows, read by the controller stage of every step tick.  The device rows are what the environments
  // run with (a write through the device pointer takes effect at the next launch), so the verbs read them back and keep no mirror.  The sensor
  // instances are twins of the applied-force instances (env_rows.h)
  bool alloc_sensors() {   // zero rows with the identity mount, generator rows seeded as seed_sensors(0, all)
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    std::vector<real> rows((size_t)n * SN_W, real(0)); std::vector<int> rng((size_t)n * SR_W, 0);
    for (int e = 0; e < n; e++) { rows[(size_t)e * SN_W + SN_QUAT] = 1; rng[(size_t)e * SR_W] = e; }
    real *r = nullptr; int *g = nullptr;
    CUDA_OK(cudaMalloc(&r, sizeof(real) * n * SN_W)); CUDA_OK(cudaMalloc(&g, sizeof(int) * n * SR_W));
    A.sn.rows = r; A.sn.rng = g;
    CUDA_OK(cudaMemcpy(r, rows.data(), sizeof(real) * n * SN_W, cudaMemcpyHostToDevice)); CUDA_OK(cudaMemcpy(g, rng.data(), sizeof(int) * n * SR_W, cudaMemcpyHostToDevice));
    return rows_rule(own, R_SN);
  }
  bool set_env_sensors(const double *enc_offset, const double *enc_noise, const double *imu_quat, const double *imu_bias, const double *imu_noise, const unsigned char *mask) override {
    const std::string verb = "cassie_batch_set_env_sensors: ";
    if (A.trace.rows) { set_err(verb + "the batch has a per-tick trace (cassie_batch_set_trace); sensor models and a trace do not combine"); return false; }
    if (A.cl.rows) { set_err(verb + "the batch has contact lists (cassie_batch_enable_contacts); sensor models and contact lists do not combine"); return false; }
    static const char *const bias_name[2] = {"gyro bias", "accelerometer bias"}, *const std_name[3] = {"orientation noise", "gyro noise", "accelerometer noise"};
    for (int e = 0; e < n; e++) {   // every masked value first
      if (mask && !mask[e]) continue;
      const std::string env = verb + "environment " + std::to_string(e) + ", ";
      for (int c = 0; c < 16; c++) {
        if (enc_offset && !std::isfinite(enc_offset[(size_t)e * 16 + c])) { set_err(env + "encoder " + std::to_string(c) + ": the offset is not finite"); return false; }
        if (enc_noise && !(std::isfinite(enc_noise[(size_t)e * 16 + c]) && enc_noise[(size_t)e * 16 + c] >= 0)) { set_err(env + "encoder " + std::to_string(c) + ": the noise std must be finite and >= 0"); return false; }
      }
      if (imu_quat) {
        const double *q = imu_quat + (size_t)e * 4; double nn = 0;
        for (int k = 0; k < 4; k++) { if (!std::isfinite(q[k])) { set_err(env + "IMU mount: quaternion component " + std::to_string(k) + " is not finite"); return false; } nn += q[k] * q[k]; }
        if (!(nn > 0)) { set_err(env + "IMU mount: the quaternion is zero"); return false; }
      }
      for (int c = 0; imu_bias && c < 6; c++) if (!std::isfinite(imu_bias[(size_t)e * 6 + c])) { set_err(env + bias_name[c / 3] + " " + "xyz"[c % 3] + ": not finite"); return false; }
      for (int c = 0; imu_noise && c < 9; c++) { const double v = imu_noise[(size_t)e * 9 + c]; if (!(std::isfinite(v) && v >= 0)) { set_err(env + std_name[c / 3] + " " + "xyz"[c % 3] + ": the std must be finite and >= 0"); return false; } }
    }
    if (!A.sn.rows && !alloc_sensors()) return false;   // the first call: the zero model
    std::vector<real> all((size_t)n * SN_W);
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a launch in flight reads the rows
    CUDA_OK(cudaMemcpy(all.data(), A.sn.rows, sizeof(real) * n * SN_W, cudaMemcpyDeviceToHost));   // unmasked environments keep what their rows hold
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      real *r = &all[(size_t)e * SN_W];
      for (int c = 0; c < 16; c++) { if (enc_offset) r[SN_ENC_OFF + c] = (real)enc_offset[(size_t)e * 16 + c]; if (enc_noise) r[SN_ENC_STD + c] = (real)enc_noise[(size_t)e * 16 + c]; }
      if (imu_quat) { const double *q = imu_quat + (size_t)e * 4; const double nn = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]); for (int k = 0; k < 4; k++) r[SN_QUAT + k] = (real)(q[k] / nn); }
      for (int k = 0; imu_bias && k < 3; k++) { r[SN_GYRO_BIAS + k] = (real)imu_bias[(size_t)e * 6 + k]; r[SN_ACC_BIAS + k] = (real)imu_bias[(size_t)e * 6 + 3 + k]; }
      for (int k = 0; imu_noise && k < 3; k++) { r[SN_ORI_STD + k] = (real)imu_noise[(size_t)e * 9 + k]; r[SN_GYRO_STD + k] = (real)imu_noise[(size_t)e * 9 + 3 + k]; r[SN_ACC_STD + k] = (real)imu_noise[(size_t)e * 9 + 6 + k]; }
    }
    CUDA_OK(cudaMemcpy((void *)A.sn.rows, all.data(), sizeof(real) * n * SN_W, cudaMemcpyHostToDevice));
    return true;
  }
  bool get_env_sensors(double *enc_offset, double *enc_noise, double *imu_quat, double *imu_bias, double *imu_noise) override {   // the zero model without rows
    std::vector<real> all((size_t)n * SN_W, real(0));
    if (A.sn.rows) { CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaMemcpyAsync(all.data(), A.sn.rows, sizeof(real) * n * SN_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream)); }
    else for (int e = 0; e < n; e++) all[(size_t)e * SN_W + SN_QUAT] = 1;
    for (int e = 0; e < n; e++) {
      const real *r = &all[(size_t)e * SN_W];
      for (int c = 0; c < 16; c++) { if (enc_offset) enc_offset[(size_t)e * 16 + c] = (double)r[SN_ENC_OFF + c]; if (enc_noise) enc_noise[(size_t)e * 16 + c] = (double)r[SN_ENC_STD + c]; }
      for (int k = 0; imu_quat && k < 4; k++) imu_quat[(size_t)e * 4 + k] = (double)r[SN_QUAT + k];
      for (int k = 0; imu_bias && k < 3; k++) { imu_bias[(size_t)e * 6 + k] = (double)r[SN_GYRO_BIAS + k]; imu_bias[(size_t)e * 6 + 3 + k] = (double)r[SN_ACC_BIAS + k]; }
      for (int k = 0; imu_noise && k < 3; k++) { imu_noise[(size_t)e * 9 + k] = (double)r[SN_ORI_STD + k]; imu_noise[(size_t)e * 9 + 3 + k] = (double)r[SN_GYRO_STD + k]; imu_noise[(size_t)e * 9 + 6 + k] = (double)r[SN_ACC_STD + k]; }
    }
    return true;
  }
  bool clear_env_sensors() override {   // back to the instances that ran before
    if (!A.sn.rows) return true;
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaFree((void *)A.sn.rows)); CUDA_OK(cudaFree(A.sn.rng)); A.sn = SensorArgs<real>{};
    return rows_rule(dropped, R_SN);
  }
  bool seed_sensors(unsigned long long seed, const unsigned char *mask) override {
    if (!A.sn.rows) { set_err("cassie_batch_seed_sensors: no sensor models (cassie_batch_set_env_sensors)"); return false; }
    std::vector<int> g((size_t)n * SR_W);
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaMemcpy(g.data(), A.sn.rng, sizeof(int) * n * SR_W, cudaMemcpyDeviceToHost));
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      const unsigned long long k = seed + (unsigned long long)e;
      g[(size_t)e * SR_W] = (int)(uint32_t)k; g[(size_t)e * SR_W + 1] = (int)(uint32_t)(k >> 32); g[(size_t)e * SR_W + 2] = 0; g[(size_t)e * SR_W + 3] = 0;
    }
    CUDA_OK(cudaMemcpy(A.sn.rng, g.data(), sizeof(int) * n * SR_W, cudaMemcpyHostToDevice));
    return true;
  }
  bool get_sensor_rng(unsigned long long *seed, unsigned long long *counter) override {
    if (!A.sn.rows) { set_err("cassie_batch_get_sensor_rng: no sensor models (cassie_batch_set_env_sensors)"); return false; }
    std::vector<int> g((size_t)n * SR_W);
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaMemcpyAsync(g.data(), A.sn.rng, sizeof(int) * n * SR_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) {
      const uint32_t *w = reinterpret_cast<const uint32_t *>(&g[(size_t)e * SR_W]);
      if (seed) seed[e] = (unsigned long long)w[0] | ((unsigned long long)w[1] << 32);
      if (counter) counter[e] = (unsigned long long)w[2] | ((unsigned long long)w[3] << 32);
    }
    return true;
  }
  bool geom_table() {   // d_gtab: device geom -> model geom, for the contact lists and the camera geom ids
    if (d_gtab) return true;
    int tab[MGT]; for (int k = 0; k < MGT; k++) tab[k] = -1;
    for (int g = 0; g < hm.ngeom && g < 256; g++) if (geom_dev[g] >= 0 && geom_dev[g] < MGT) tab[geom_dev[g]] = g;
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMalloc(&d_gtab, sizeof tab)); CUDA_OK(cudaMemcpy(d_gtab, tab, sizeof tab, cudaMemcpyHostToDevice));
    return true;
  }
  bool get_contacts(double *out) override {
    if (!A.cl.rows) { set_err("cassie_batch_get_contacts: no contact-list rows (cassie_batch_enable_contacts)"); return false; }
    if (!out) { set_err("cassie_batch_get_contacts: out is required"); return false; }
    return d2h(A.cl.rows, CON_W, CON_W, 0, out);
  }
  int trace_width() const override { return A.trace.T * A.trace.k; }
  // ---- the controller-stage state: the delay line, the encoders' filters (views of the cst / dfilt rows; snapshots carry them)
  bool get_actuator_state(double *torque_delay, int *drive_filter, double *joint_x, double *joint_y) override {
    CUDA_OK(cudaSetDevice(device));
    std::vector<real> cst; std::vector<int> df;   // only the rows asked for are downloaded
    if (torque_delay || joint_x || joint_y) { cst.resize((size_t)n * CST_W); CUDA_OK(cudaMemcpyAsync(cst.data(), A.cst, sizeof(real) * n * CST_W, cudaMemcpyDeviceToHost, stream)); }
    if (drive_filter) { df.resize((size_t)n * DFILT_W); CUDA_OK(cudaMemcpyAsync(df.data(), A.dfilt, sizeof(int) * n * DFILT_W, cudaMemcpyDeviceToHost, stream)); }
    CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) {
      const real *c = cst.empty() ? nullptr : &cst[(size_t)e * CST_W];
      if (torque_delay) for (int i = 0; i < 60; i++) torque_delay[(size_t)e * 60 + i] = (double)c[CS_DELAY + i];
      if (joint_x) for (int i = 0; i < 24; i++) joint_x[(size_t)e * 24 + i] = (double)c[CS_JFX + i];
      if (joint_y) for (int i = 0; i < 18; i++) joint_y[(size_t)e * 18 + i] = (double)c[CS_JFY + i];
      if (drive_filter) memcpy(drive_filter + (size_t)e * 90, &df[(size_t)e * DFILT_W], sizeof(int) * 90);
    }
    return true;
  }
  bool set_actuator_state(const double *torque_delay, const int *drive_filter, const double *joint_x, const double *joint_y, const unsigned char *mask) override {
    CUDA_OK(cudaSetDevice(device));
    std::vector<real> cst((size_t)n * CST_W); std::vector<int> df((size_t)n * DFILT_W);
    CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaMemcpy(cst.data(), A.cst, sizeof(real) * n * CST_W, cudaMemcpyDeviceToHost));
    CUDA_OK(cudaMemcpy(df.data(), A.dfilt, sizeof(int) * n * DFILT_W, cudaMemcpyDeviceToHost));
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      real *c = &cst[(size_t)e * CST_W];
      if (torque_delay) for (int i = 0; i < 60; i++) c[CS_DELAY + i] = (real)torque_delay[(size_t)e * 60 + i];
      if (joint_x) for (int i = 0; i < 24; i++) c[CS_JFX + i] = (real)joint_x[(size_t)e * 24 + i];
      if (joint_y) for (int i = 0; i < 18; i++) c[CS_JFY + i] = (real)joint_y[(size_t)e * 18 + i];
      if (drive_filter) memcpy(&df[(size_t)e * DFILT_W], drive_filter + (size_t)e * 90, sizeof(int) * 90);
    }
    if (torque_delay || joint_x || joint_y) CUDA_OK(cudaMemcpy(A.cst, cst.data(), sizeof(real) * n * CST_W, cudaMemcpyHostToDevice));
    if (drive_filter) CUDA_OK(cudaMemcpy(A.dfilt, df.data(), sizeof(int) * n * DFILT_W, cudaMemcpyHostToDevice));
    return true;
  }
  // ---- frame rows: the table is checked as a whole before anything changes; the rows start at zero and are filled by the next step / forward launch
  bool set_frames(const char *const *names, const int *kinds, int count) override {
    if (count < 0 || count > FRAME_MAX || (count > 0 && (!names || !kinds))) { set_err("cassie_batch_set_frames: between 0 and " + std::to_string(FRAME_MAX) + " frames, with names and kinds"); return false; }
    if ((A.trace.need >> TC_FRAME) & 1) { set_err("cassie_batch_set_frames: a traced column reads the frame rows (cassie_batch_set_trace)"); return false; }
    std::vector<real> tab((size_t)count * FT_W); std::vector<int> list;
    for (int f = 0; f < count; f++) {
      std::string err; const int id = frame_table_row(hm, names[f], kinds[f], &tab[(size_t)f * FT_W], err);
      if (id < 0) { set_err("cassie_batch_set_frames: " + err); return false; }
      list.push_back(kinds[f]); list.push_back(id);
    }
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    const bool acc_on = A.acc != nullptr;
    CUDA_OK(cudaFree(A.frames)); CUDA_OK(cudaFree((void *)A.ftab)); CUDA_OK(cudaFree(A.acc)); A.frames = nullptr; A.ftab = nullptr; A.acc = nullptr; A.nfr = 0; frame_list.clear();
    if (count > 0) {
      real *t = nullptr;
      CUDA_OK(cudaMalloc(&t, sizeof(real) * tab.size())); A.ftab = t;
      CUDA_OK(cudaMemcpy(t, tab.data(), sizeof(real) * tab.size(), cudaMemcpyHostToDevice));
      CUDA_OK(cudaMalloc(&A.frames, sizeof(real) * n * count * FRAME_W)); CUDA_OK(cudaMemset(A.frames, 0, sizeof(real) * n * count * FRAME_W));
      A.nfr = count; frame_list = list;
    }
    return !acc_on || enable_accelerations(true);   // the acceleration rows follow the new frame list: its width, zero until the next launch
  }
  // ---- acceleration rows (qacc and the cacc of every frame), filled by every step / forward launch from then on
  bool enable_accelerations(bool on) override {
    CUDA_OK(cudaSetDevice(device));
    const size_t bytes = sizeof(real) * n * acc_width(A.nfr);
    if (on && !A.acc) { CUDA_OK(cudaMalloc(&A.acc, bytes)); CUDA_OK(cudaMemsetAsync(A.acc, 0, bytes, stream)); CUDA_OK(cudaStreamSynchronize(stream)); }
    if (!on && A.acc) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(A.acc)); A.acc = nullptr; }
    return true;
  }
  bool get_accelerations(double *qacc, double *cacc) override {
    if (!A.acc) { set_err("cassie_batch_get_accelerations: no acceleration rows (cassie_batch_enable_accelerations)"); return false; }
    const int w = acc_width(A.nfr), nv = hm.nv;
    CUDA_OK(cudaSetDevice(device));
    h_tmp.resize((size_t)n * w);
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), A.acc, sizeof(real) * n * w, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) {
      const real *r = &h_tmp[(size_t)e * w];
      if (qacc) for (int i = 0; i < nv; i++) qacc[(size_t)e * nv + i] = (double)r[AC_QACC + i];
      if (cacc) for (int f = 0; f < A.nfr; f++) for (int k = 0; k < 6; k++) cacc[((size_t)e * A.nfr + f) * 6 + k] = (double)r[AC_CACC + AC_SLOT * f + k];
    }
    return true;
  }
  // the Jacobian of frame `frame` at the current state of every environment: one mode-4 launch (kinematics and centre of mass only, nothing else
  // written), then a synchronous copy; the Jacobian rows are allocated on first use
  bool frame_jacobian(int frame, double *jacp, double *jacr) override {
    if (frame < 0 || frame >= A.nfr) { set_err("cassie_batch_frame_jacobian: frame " + std::to_string(frame) + " of " + std::to_string(A.nfr)); return false; }
    if (!jacp) { set_err("cassie_batch_frame_jacobian: jacp is required"); return false; }
    CUDA_OK(cudaSetDevice(device));
    if (!A.jac) { CUDA_OK(cudaMalloc(&A.jac, sizeof(real) * n * FRAME_JAC_W)); CUDA_OK(cudaMemsetAsync(A.jac, 0, sizeof(real) * n * FRAME_JAC_W, stream)); }
    A.jfr = frame;
    if (!step(0, 4)) return false;
    h_tmp.resize((size_t)n * FRAME_JAC_W);
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), A.jac, sizeof(real) * n * FRAME_JAC_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    const int nv = hm.nv;
    for (int e = 0; e < n; e++) for (int k = 0; k < 3; k++) for (int j = 0; j < nv; j++) {
      const real *r = &h_tmp[(size_t)e * FRAME_JAC_W];
      jacp[((size_t)e * 3 + k) * nv + j] = (double)r[k * FJ_COLS + j];
      if (jacr) jacr[((size_t)e * 3 + k) * nv + j] = (double)r[(3 + k) * FJ_COLS + j];
    }
    return true;
  }
  // dynamics at the current state of every environment: one mode-5 launch on the batch stream (kinematics, centre of mass, CRB and the bias forces;
  // nothing else written).  The rows are allocated on first use; snapshots and resets leave them alone (a query result, not state).
  bool dynamics() override {
    CUDA_OK(cudaSetDevice(device));
    if (!A.dyn) CUDA_OK(cudaMalloc(&A.dyn, sizeof(real) * n * DYN_W));
    if (!step(0, 5)) return false;
    dyn_done = true;
    return true;
  }
  bool get_dynamics(double *M, double *bias, double *J_eq, double *eq_err, double *Icm) override {
    if (!dyn_done) { set_err("cassie_batch_get_dynamics: no dynamics launch yet (cassie_batch_dynamics)"); return false; }
    CUDA_OK(cudaSetDevice(device));
    h_tmp.resize((size_t)n * DYN_W);
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), A.dyn, sizeof(real) * n * DYN_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    const int nv = hm.nv, ne = 3 * hm.neq;
    for (int e = 0; e < n; e++) {
      const real *r = &h_tmp[(size_t)e * DYN_W];
      if (M) for (int i = 0; i < nv; i++) for (int j = 0; j < nv; j++) M[((size_t)e * nv + i) * nv + j] = (double)r[DY_M + i * DY_COLS + j];
      if (bias) for (int i = 0; i < nv; i++) bias[(size_t)e * nv + i] = (double)r[DY_BIAS + i];
      if (J_eq) for (int i = 0; i < ne; i++) for (int j = 0; j < nv; j++) J_eq[((size_t)e * ne + i) * nv + j] = (double)r[DY_JEQ + i * DY_COLS + j];
      if (eq_err) for (int i = 0; i < ne; i++) eq_err[(size_t)e * ne + i] = (double)r[DY_EQPOS + i];
      if (Icm) centroid_inertia(r, &Icm[(size_t)e * 9]);
    }
    return true;
  }
  // inverse dynamics at the current state of every environment and the qacc of the inverse-input rows: one mode-6 launch on the batch stream.  The input
  // and output rows and the launch's scratch rows are allocated (the rows zeroed) on first use, by this or by the device pointers, freed with the batch;
  // snapshots and resets leave them alone.
  bool alloc_inverse() {
    CUDA_OK(cudaSetDevice(device));
    if (d_iq) return true;
    CUDA_OK(cudaMalloc(&d_iq, sizeof(real) * n * VW)); CUDA_OK(cudaMemsetAsync(d_iq, 0, sizeof(real) * n * VW, stream));
    CUDA_OK(cudaMalloc(&A.inv, sizeof(real) * n * INV_W)); CUDA_OK(cudaMemsetAsync(A.inv, 0, sizeof(real) * n * INV_W, stream));
    CUDA_OK(cudaMalloc(&d_idbg, sizeof(real) * n * D_SIZE)); CUDA_OK(cudaMalloc(&d_icst, sizeof(real) * n * CST_W));
    CUDA_OK(cudaMalloc(&d_icnt, sizeof(int) * n * 8)); CUDA_OK(cudaMemsetAsync(d_icnt, 0, sizeof(int) * n * 8, stream));
    CUDA_OK(cudaStreamSynchronize(stream));   // zeroed before a caller writes the input rows on another stream
    return true;
  }
  bool inverse(const double *qacc) override {
    if (!qacc && !d_iq) { set_err("cassie_batch_inverse: no qacc: pass one, or write the rows of cassie_batch_device_ptr(b, \"inv_qacc\") first"); return false; }
    if (!alloc_inverse()) return false;
    if (qacc) {
      const int nv = hm.nv;
      h_tmp.assign((size_t)n * VW, 0);
      for (int e = 0; e < n; e++) for (int i = 0; i < nv; i++) h_tmp[(size_t)e * VW + i] = (real)qacc[(size_t)e * nv + i];   // column = dof (the extra body at 32..37)
      CUDA_OK(cudaMemcpyAsync(d_iq, h_tmp.data(), sizeof(real) * n * VW, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    }
    if (!step(0, 6)) return false;
    inv_done = true;
    return true;
  }
  bool get_inverse(double *qfrc_inverse, double *qfrc_constraint, int *counts) override {
    if (!inv_done) { set_err("cassie_batch_get_inverse: no inverse launch yet (cassie_batch_inverse)"); return false; }
    CUDA_OK(cudaSetDevice(device));
    h_tmp.resize((size_t)n * INV_W);
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), A.inv, sizeof(real) * n * INV_W, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    const int nv = hm.nv;
    for (int e = 0; e < n; e++) {
      const real *r = &h_tmp[(size_t)e * INV_W];
      if (qfrc_inverse) for (int i = 0; i < nv; i++) qfrc_inverse[(size_t)e * nv + i] = (double)r[IV_QFRC + i];
      if (qfrc_constraint) for (int i = 0; i < nv; i++) qfrc_constraint[(size_t)e * nv + i] = (double)r[IV_QFRCC + i];
      if (counts) { counts[3 * e] = (int)r[IV_NEFC]; counts[3 * e + 1] = (int)r[IV_NCON]; counts[3 * e + 2] = (int)r[IV_DROPPED]; }
    }
    return true;
  }
  bool set_rays(const int *frame, const double *origin, const double *dir, const double *max_dist, int k) override {
    std::vector<double> tab; std::string err;
    if (!ray_table(frame, origin, dir, max_dist, k, tab, err)) { set_err("cassie_batch_set_rays: " + err); return false; }
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaFree(d_rtab)); CUDA_OK(cudaFree(d_rays)); d_rtab = d_rays = nullptr; nray = 0; rays_done = false;
    if (k == 0) return true;
    std::vector<real> t(tab.begin(), tab.end());
    CUDA_OK(cudaMalloc(&d_rtab, sizeof(real) * t.size())); CUDA_OK(cudaMemcpy(d_rtab, t.data(), sizeof(real) * t.size(), cudaMemcpyHostToDevice));
    nray = k;
    return true;
  }
  bool raycast() override {
    if (!nray) { set_err("cassie_batch_raycast: no rays are set (cassie_batch_set_rays)"); return false; }
    CUDA_OK(cudaSetDevice(device));
    if (!d_rays) CUDA_OK(cudaMalloc(&d_rays, sizeof(real) * n * nray * RAY_SLOT));
    RayArgs<real> R; R.model = d_model; R.qpos = A.qpos; R.qpos_w = QW; R.genv = d_genv; R.hfield = A.hfield; R.n_terrain = A.n_terrain; R.hfield_stride = A.hfield_stride; R.terrain = d_terrain; R.bpos = A.bpos;
    R.tab = d_rtab; R.k = nray; R.out = d_rays; R.n = n;
    CUDA_OK(launch_raycast<real>(R, device, stream));
    launches++; rays_done = true;
    return true;
  }
  bool get_rays(double *out) override {
    if (!rays_done) { set_err("cassie_batch_get_rays: no cast since the rays were set (cassie_batch_raycast)"); return false; }
    if (!out) { set_err("cassie_batch_get_rays: out is required"); return false; }
    return d2h(d_rays, nray * RAY_SLOT, nray * RAY_SLOT, 0, out);
  }
  bool set_cameras(int k, const int *body, const double *pos, const double *quat, const double *fovy, int width, int height, double zfar, const char *verb,
                   bool indexed) override {
    Cameras c; std::string err;
    if (k < 0 || k > CAM_MAX) { set_err(std::string(verb) + ": between 0 and " + std::to_string(CAM_MAX) + " cameras"); return false; }
    if (k > 0 && (!body || !pos || !quat || !fovy)) { set_err(std::string(verb) + ": body, pos, quat and fovy are required"); return false; }
    for (int i = 0; i < k; i++) {
      const std::string at = std::string(verb) + (indexed ? ": camera " + std::to_string(i) : "");
      if (body[i] < 0 || body[i] >= hm.nbody) { set_err(at + ": unknown body"); return false; }
      if (!camera_check(pos + 3 * i, quat + 4 * i, fovy[i], width, height, zfar, c.quat[i], err)) { set_err(at + ": " + err); return false; }
      c.body[i] = body[i]; c.fovy[i] = fovy[i];
      for (int j = 0; j < 3; j++) c.pos[i][j] = pos[3 * i + j];
    }
    if (k > 0) { c.k = k; c.width = width; c.height = height; c.zfar = zfar; }
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaFree(d_depth)); CUDA_OK(cudaFree(d_camgeom)); CUDA_OK(cudaFree(d_camenv)); d_depth = nullptr; d_camgeom = nullptr; d_camenv = nullptr;
    ce_host.clear(); depth_done = geoms_done = false;
    cam = c;
    return true;
  }
  bool render_depth() override {
    if (!cam.k) { set_err("cassie_batch_render_depth: no camera is set (cassie_batch_set_camera)"); return false; }
    CUDA_OK(cudaSetDevice(device));
    const size_t px = (size_t)n * cam.k * cam.width * cam.height;
    if (!d_depth) CUDA_OK(cudaMalloc(&d_depth, sizeof(real) * px));
    if (cam_geoms && !d_camgeom) { if (!geom_table()) return false; CUDA_OK(cudaMalloc(&d_camgeom, sizeof(int) * px)); }
    CamMount<real> mt[CAM_MAX];
    for (int c = 0; c < cam.k; c++) {
      mt[c].body = cam.body[c]; mt[c].tan_half = (real)std::tan(cam.fovy[c] * M_PI / 360);
      for (int i = 0; i < 3; i++) mt[c].pos[i] = (real)cam.pos[c][i];
      for (int i = 0; i < 4; i++) mt[c].quat[i] = (real)cam.quat[c][i];
    }
    if (cam.k == 1 && !d_camenv && !cam_geoms) {   // one camera, nothing per environment: the one-camera kernel (DESIGN.md section 5)
      CamArgs<real> C; C.model = d_model; C.qpos = A.qpos; C.qpos_w = QW; C.genv = d_genv; C.hfield = A.hfield; C.n_terrain = A.n_terrain; C.hfield_stride = A.hfield_stride; C.terrain = d_terrain; C.bpos = A.bpos;
      C.body = mt[0].body; C.width = cam.width; C.height = cam.height; C.tan_half = mt[0].tan_half; C.zfar = (real)cam.zfar;
      for (int i = 0; i < 3; i++) C.pos[i] = mt[0].pos[i];
      for (int i = 0; i < 4; i++) C.quat[i] = mt[0].quat[i];
      C.out = d_depth; C.n = n;
      CUDA_OK(launch_camera<real>(C, device, stream));
    } else {
      CamSetArgs<real> C; C.model = d_model; C.qpos = A.qpos; C.qpos_w = QW; C.genv = d_genv; C.hfield = A.hfield; C.n_terrain = A.n_terrain; C.hfield_stride = A.hfield_stride; C.terrain = d_terrain; C.bpos = A.bpos;
      C.k = cam.k; C.width = cam.width; C.height = cam.height; C.zfar = (real)cam.zfar;
      for (int c = 0; c < CAM_MAX; c++) C.cam[c] = mt[c < cam.k ? c : 0];
      C.out = d_depth; C.n = n; C.cenv = d_camenv; C.geom = cam_geoms ? d_camgeom : nullptr; C.gtab = d_gtab;
      CUDA_OK(launch_camera_set<real>(C, device, stream));
    }
    launches++; depth_done = true; geoms_done = cam_geoms;
    return true;
  }
  bool get_depth(double *out) override {
    if (!depth_done) { set_err("cassie_batch_get_depth: no render since the camera was set (cassie_batch_render_depth)"); return false; }
    if (!out) { set_err("cassie_batch_get_depth: out is required"); return false; }
    const int w = cam.k * cam.width * cam.height;
    return d2h(d_depth, w, w, 0, out);
  }
  bool enable_camera_geoms(bool on) override {
    if (on == cam_geoms) return true;
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a render in flight writes the rows
    CUDA_OK(cudaFree(d_camgeom)); d_camgeom = nullptr;
    cam_geoms = on; geoms_done = false;
    return true;
  }
  bool get_camera_geoms(int *out) override {
    if (!geoms_done) { set_err("cassie_batch_get_camera_geoms: no render with geom ids since the cameras were set or geom ids enabled (cassie_batch_enable_camera_geoms, cassie_batch_render_depth)"); return false; }
    if (!out) { set_err("cassie_batch_get_camera_geoms: out is required"); return false; }
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(out, d_camgeom, sizeof(int) * n * cam.k * cam.width * cam.height, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  // ---- per-environment camera mounts (extrinsics and field-of-view randomisation): the pose in each camera's body frame and its fovy, per
  // environment; the body stays the set's.  As with the actuator rows, the device rows are what the kernel reads, the mirror keeps the doubles the verb
  // was last given, and get reports a value the row still holds as the verb stored it as the verb was given it
  void model_camenv(int c, double *v) const { for (int i = 0; i < 3; i++) v[CE_POS + i] = cam.pos[c][i]; for (int i = 0; i < 4; i++) v[CE_QUAT + i] = cam.quat[c][i]; v[CE_FOVY] = cam.fovy[c]; }
  bool pull_camenv(std::vector<real> &all) {
    const size_t w = (size_t)n * cam.k * CAMENV_SLOT;
    all.assign(w, real(0));
    if (!d_camenv) return true;
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(all.data(), d_camenv, sizeof(real) * w, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  bool set_env_cameras(const double *pos, const double *quat, const double *fovy, const unsigned char *mask) override {
    const std::string verb = "cassie_batch_set_env_cameras";
    const int k = cam.k;
    if (!k) { set_err(verb + ": no cameras are set (cassie_batch_set_cameras)"); return false; }
    for (int e = 0; e < n; e++) {   // every masked value is checked before anything changes
      if (mask && !mask[e]) continue;
      for (int c = 0; c < k; c++) {
        const size_t i = (size_t)e * k + c; const std::string at = verb + ": environment " + std::to_string(e) + ", camera " + std::to_string(c) + ": ";
        if (pos && !std::isfinite(pos[3 * i] + pos[3 * i + 1] + pos[3 * i + 2])) { set_err(at + "pos must be finite"); return false; }
        if (quat) {
          const double *q = quat + 4 * i, nq = std::sqrt(q[0] * q[0] + q[1] * q[1] + q[2] * q[2] + q[3] * q[3]);
          if (!(nq > 0) || !std::isfinite(nq)) { set_err(at + "quat must be finite and non-zero"); return false; }
        }
        if (fovy && !(fovy[i] > 0 && fovy[i] < 180)) { set_err(at + "fovy must be in (0, 180) degrees"); return false; }
      }
    }
    std::vector<real> all;
    if (!d_camenv) {   // the first call: every environment starts from the set's mounts
      ce_host.resize((size_t)n * k * CAMENV_SLOT); all.resize(ce_host.size());
      for (int e = 0; e < n; e++) for (int c = 0; c < k; c++) model_camenv(c, &ce_host[((size_t)e * k + c) * CAMENV_SLOT]);
      for (size_t i = 0; i < all.size(); i++) all[i] = (real)ce_host[i];
    } else if (!pull_camenv(all)) return false;   // unmasked environments keep what their rows hold, also when it was written on the device
    for (int e = 0; e < n; e++) {
      if (mask && !mask[e]) continue;
      for (int c = 0; c < k; c++) {
        const size_t i = (size_t)e * k + c; double *h = &ce_host[i * CAMENV_SLOT]; real *r = &all[i * CAMENV_SLOT];
        if (pos) for (int j = 0; j < 3; j++) { h[CE_POS + j] = pos[3 * i + j]; r[CE_POS + j] = (real)h[CE_POS + j]; }
        if (quat) for (int j = 0; j < 4; j++) { h[CE_QUAT + j] = quat[4 * i + j]; r[CE_QUAT + j] = (real)h[CE_QUAT + j]; }
        if (fovy) { h[CE_FOVY] = fovy[i]; r[CE_FOVY] = (real)h[CE_FOVY]; }
      }
    }
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));   // a render in flight reads the rows
    if (!d_camenv) CUDA_OK(cudaMalloc(&d_camenv, sizeof(real) * all.size()));
    CUDA_OK(cudaMemcpy(d_camenv, all.data(), sizeof(real) * all.size(), cudaMemcpyHostToDevice));
    return true;
  }
  bool get_env_cameras(double *pos, double *quat, double *fovy) override {
    const int k = cam.k;
    if (!k) { set_err("cassie_batch_get_env_cameras: no cameras are set (cassie_batch_set_cameras)"); return false; }
    std::vector<real> all;
    if (!pull_camenv(all)) return false;
    for (int e = 0; e < n; e++) for (int c = 0; c < k; c++) {
      const size_t i = (size_t)e * k + c; double v[CAMENV_SLOT];
      model_camenv(c, v);
      if (d_camenv) for (int f = 0; f < CAMENV_SLOT; f++) {
        const double h = ce_host[i * CAMENV_SLOT + f]; const real dv = all[i * CAMENV_SLOT + f];
        v[f] = dv == (real)h ? h : (double)dv;
      }
      if (pos) for (int j = 0; j < 3; j++) pos[3 * i + j] = v[CE_POS + j];
      if (quat) for (int j = 0; j < 4; j++) quat[4 * i + j] = v[CE_QUAT + j];
      if (fovy) fovy[i] = v[CE_FOVY];
    }
    return true;
  }
  bool clear_env_cameras() override {   // back to the set's mounts
    ce_host.clear();
    if (!d_camenv) return true;
    CUDA_OK(cudaSetDevice(device)); CUDA_OK(cudaStreamSynchronize(stream));
    CUDA_OK(cudaFree(d_camenv)); d_camenv = nullptr;
    return true;
  }
  // open-loop sinusoidal gait on the motor-PD targets (BASELINE config 5 "random PD gaits"): evaluated in the kernel every control tick, so
  // multi-tick launches follow it without a host round trip; installing it restarts the tick clock
  bool set_pd_gait(const double *amp, const double *freq, const double *phase) override {
    CUDA_OK(cudaSetDevice(device));
    if (!amp || !freq || !phase) { if (A.gait) { CUDA_OK(cudaStreamSynchronize(stream)); CUDA_OK(cudaFree(A.gait)); A.gait = nullptr; } return true; }
    if (!A.gait) CUDA_OK(cudaMalloc(&A.gait, sizeof(real) * n * GAIT_W));
    h_tmp.assign((size_t)n * GAIT_W, 0);
    for (int e = 0; e < n; e++) { real *r = &h_tmp[(size_t)e * GAIT_W]; for (int i = 0; i < 10; i++) { r[GA_AMP + i] = (real)amp[(size_t)e * 10 + i]; r[GA_PHASE + i] = (real)phase[(size_t)e * 10 + i]; } r[GA_FREQ] = (real)freq[e]; }
    CUDA_OK(cudaMemcpyAsync(A.gait, h_tmp.data(), sizeof(real) * n * GAIT_W, cudaMemcpyHostToDevice, stream));
    CUDA_OK(cudaMemset2DAsync(A.dfilt + DF_TICK, sizeof(int) * DFILT_W, 0, sizeof(int), n, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  bool step(int nticks, int mode) override { return step_range(nticks, mode, 0, n, stream); }
  // the features a launch of `mode` asks for (devmodel.h F_*): the model's and one per kind of per-environment rows the batch holds; frame,
  // acceleration, dynamics and inverse rows: an F_FR instance (set_const launches too: they write no frames)
  int launch_feat(int mode) const {
    return (A.genv ? feat | F_EG : feat) | (A.terrain ? F_TR : 0) | (A.bpos ? F_BP : 0) | (A.act ? F_AC : 0) | (A.mech ? F_MC : 0) | (A.contact ? F_CT : 0) | (A.applied ? F_XF : 0) |
           (A.trace.rows ? F_TC : 0) | (A.cl.rows ? F_CL : 0) | (A.sn.rows ? F_SN : 0) | ((A.frames || A.acc || A.cl.rows || mode == 5 || mode == 6) ? F_FR : 0);
  }
  // the instance kind a launch of `mode` runs: 0 plain, 1 extended, 2 plain + estimator
  int launch_kind(int mode) {
    // per-environment model constants / derived-quantity rows / task-space PD / set_const: extended instance (its own scratch size and launch shape);
    // the in-kernel estimator alone: the plain instance with the estimator stage
    const int ext = (A.cenv || A.aux || A.task || A.frames || A.acc || A.trace.rows || A.cl.rows || (A.dbg && !DBG_IN_ALL_INSTANCES) || mode >= 3) ? 1 : (A.est ? 2 : 0);   // debug batches: the stage dumps live in the extended instance
    return select_step<real>(ext, launch_feat(mode)).kind;   // applied forces: a plain twin where f04 / f24 would run, else the extended kind
  }
  bool step_range(int nticks, int mode, int env0, int count, cudaStream_t on) {   // the launch covers environments [env0, env0 + count)
    CUDA_OK(cudaSetDevice(device));
    if (mode == 2 && !A.aux) { set_err("query needs the derived-quantity rows (cassie_batch_enable_aux)"); return false; }
    if (mode == 4 && (!A.frames || !A.jac)) { set_err("the frame Jacobian needs frames (cassie_batch_set_frames)"); return false; }
    if (mode == 5 && !A.dyn) { set_err("the dynamics launch needs its rows (cassie_batch_dynamics)"); return false; }
    if (mode == 6 && !d_iq) { set_err("the inverse launch needs its rows (cassie_batch_inverse)"); return false; }
    A.nsub = nsub_override;
    const int ext = launch_kind(mode);
    if (!rows_rule(lend_for_launch, ext)) return false;   // rows a verb dropped since their holder's set, and the extended chain twins' contact rows
    A.warp_stride = (int)warp_bytes<real>(A.ystride, ext == 1);
    const LaunchCfg &c = cfg[ext];
    int grid = (count + c.wpb - 1) / c.wpb; if (grid > c.resident_ctas) grid = c.resident_ctas;
    EnvArrays<real> La = A; La.env0 = env0; La.n = count;   // the argument block of this launch
    if (mode == 5 || mode == 6) La.dbg = nullptr;   // the dynamics and inverse launches write their rows only, also in a debug batch
    // mode 6: the caller's qacc reaches the lanes through the warm-start load (mode 6 writes no state back); the forward's stage dump, sensor data and
    // counters go to the launch's scratch rows, for inverse_row; no aux or frame rows
    if (mode == 6) { La.qacc_ws = d_iq; La.dbg = d_idbg; La.cst = d_icst; La.counters = d_icnt; La.aux = nullptr; La.nfr = 0; }
    const StepChoice inst = select_step<real>(ext, launch_feat(mode));   // with the rows provisioned above
    if (inst.kind != ext || inst.index < 0) { set_err("no step-kernel instance is compiled for this batch's rows"); return false; }
    { const DevModel<real> *dm = d_model; void *args[4] = {(void *)&dm, (void *)&La, (void *)&nticks, (void *)&mode};
      CUDA_OK(cudaLaunchKernel(STEP_INSTANCES[inst.index].entry(), dim3(grid), dim3(32 * c.wpb), args, c.smem, on)); }
    launches++;
    if (mode == 0 && A.trace.rows) tc_ticks = nticks < A.trace.T ? nticks : A.trace.T;
    CUDA_OK(cudaGetLastError());
    return true;
  }
  bool integrate() override {
    CUDA_OK(cudaSetDevice(device));
    const int ntiles = (n + ITILE - 1) / ITILE; int sms = 0; CUDA_OK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, device));
    const size_t ib = ISTAGES * itile_bytes<real>(A.qpos_w, A.qvel_w);
    CUDA_OK(cudaFuncSetAttribute(cassie_integrate_kernel<real>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)ib));
    const int per_sm = (int)(220000 / ib) < 1 ? 1 : (int)(220000 / ib);
    const int grid = ntiles < sms * per_sm ? ntiles : sms * per_sm;
    cassie_integrate_kernel<real><<<grid, 256, ib, stream>>>(d_model, A.qpos, A.qvel, n, A.qpos_w, A.qvel_w);
    launches++;
    CUDA_OK(cudaGetLastError());
    return true;
  }
  bool d2h(const real *src, int w, int take, int off, double *out) {
    h_tmp.resize((size_t)n * w);
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), src, sizeof(real) * n * w, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) for (int i = 0; i < take; i++) out[(size_t)e * take + i] = (double)h_tmp[(size_t)e * w + off + i];
    return true;
  }
  bool get(const char *f, double *out) override {
    if (!strcmp(f, "qpos")) return d2h(A.qpos, QW, hm.nq, 0, out);
    if (!strcmp(f, "qvel")) return d2h(A.qvel, VW, hm.nv, 0, out);
    if (!strcmp(f, "qacc_ws")) return d2h(A.qacc_ws, VW, hm.nv, 0, out);
    if (!strcmp(f, "time")) return d2h(A.cst, CST_W, 1, CS_TIME, out);
    if (!strcmp(f, "obs")) return d2h(A.obs, OBS_W, OBS_W, 0, out);
    if (!strcmp(f, "cst")) return d2h(A.cst, CST_W, CST_W, 0, out);
    if (!strcmp(f, "xfrc")) return d2h(A.xfrc, XFRC_W, XFRC_W, 0, out);
    if (!strcmp(f, "est_out")) { if (!A.est) { set_err("the in-kernel estimator is not enabled (cassie_batch_enable_estimator_device)"); return false; } return d2h(A.obs, OBS_W, EO_W, OB_EST_OUT, out); }
    if (!strcmp(f, "aux")) { if (!A.aux) { set_err("derived quantities are not enabled (cassie_batch_enable_aux)"); return false; } return d2h(A.aux, AUX_W, AUX_W, 0, out); }
    if (!strcmp(f, "frames")) { if (!A.frames) { set_err("no frames are set (cassie_batch_set_frames)"); return false; } return d2h(A.frames, A.nfr * FRAME_W, A.nfr * FRAME_W, 0, out); }
    if (!strcmp(f, "acc")) { if (!A.acc) { set_err("no acceleration rows (cassie_batch_enable_accelerations)"); return false; } return d2h(A.acc, acc_width(A.nfr), acc_width(A.nfr), 0, out); }
    set_err(std::string("unknown field ") + f); return false;
  }
  bool h2d(real *dst, int w, int take, int off, const double *in) {
    h_tmp.resize((size_t)n * w);
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(h_tmp.data(), dst, sizeof(real) * n * w, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    for (int e = 0; e < n; e++) for (int i = 0; i < take; i++) h_tmp[(size_t)e * w + off + i] = (real)in[(size_t)e * take + i];
    CUDA_OK(cudaMemcpyAsync(dst, h_tmp.data(), sizeof(real) * n * w, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  bool set(const char *f, const double *in) override {
    if (!strcmp(f, "qpos")) return h2d(A.qpos, QW, hm.nq, 0, in);
    if (!strcmp(f, "qvel")) return h2d(A.qvel, VW, hm.nv, 0, in);
    if (!strcmp(f, "time")) return h2d(A.cst, CST_W, 1, CS_TIME, in);
    if (!strcmp(f, "sto")) return h2d(A.cst, CST_W, 1, CS_STO, in);
    if (!strcmp(f, "cst")) return h2d(A.cst, CST_W, CST_W, 0, in);
    if (!strcmp(f, "acc")) { if (!A.acc) { set_err("no acceleration rows (cassie_batch_enable_accelerations)"); return false; } return h2d(A.acc, acc_width(A.nfr), acc_width(A.nfr), 0, in); }
    set_err(std::string("unknown field ") + f); return false;
  }
  bool set_xfrc(const double *xfrc, int body) override {
    h_tmp.assign((size_t)n * XFRC_W, 0);
    if (xfrc) for (int e = 0; e < n; e++) { for (int i = 0; i < 6; i++) h_tmp[(size_t)e * XFRC_W + i] = (real)xfrc[(size_t)e * 6 + i]; h_tmp[(size_t)e * XFRC_W + 6] = (real)body; }
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(A.xfrc, h_tmp.data(), sizeof(real) * n * XFRC_W, cudaMemcpyHostToDevice, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  void *dev_ptr(const char *f) override {
    if (!strcmp(f, "qpos")) return A.qpos; if (!strcmp(f, "qvel")) return A.qvel; if (!strcmp(f, "pd")) return A.pd; if (!strcmp(f, "obs")) return A.obs;
    if (!strcmp(f, "xfrc")) return A.xfrc; if (!strcmp(f, "cst")) return A.cst; if (!strcmp(f, "qacc_ws")) return A.qacc_ws; if (!strcmp(f, "aux")) return A.aux; if (!strcmp(f, "task")) return A.task;
    if (!strcmp(f, "frames")) return A.frames; if (!strcmp(f, "frame_jac")) return A.jac; if (!strcmp(f, "dyn")) return A.dyn; if (!strcmp(f, "acc")) return A.acc;
    if (!strcmp(f, "rays")) return d_rays; if (!strcmp(f, "depth")) return d_depth; if (!strcmp(f, "camera_env")) return d_camenv; if (!strcmp(f, "camera_geom")) return d_camgeom; if (!strcmp(f, "terrain")) return d_terrain; if (!strcmp(f, "actuators")) return row(R_ACT); if (!strcmp(f, "mechanics")) return row(R_MECH); if (!strcmp(f, "contact")) return row(R_CT);
    if (!strcmp(f, "applied")) return row(R_APP); if (!strcmp(f, "loops")) return d_loops; if (!strcmp(f, "ik_targets")) return d_ikt; if (!strcmp(f, "ik")) return d_ik;
    if (!strcmp(f, "inv_qacc") || !strcmp(f, "inv")) { if (!alloc_inverse()) return nullptr; return !strcmp(f, "inv") ? A.inv : d_iq; }
    if (!strcmp(f, "trace")) return A.trace.rows;
    if (!strcmp(f, "contacts")) return A.cl.rows;
    if (!strcmp(f, "sensors")) return (void *)A.sn.rows; if (!strcmp(f, "sensor_rng")) return A.sn.rng;
#ifdef CASSIE_STAGE_CLOCKS
    if (!strcmp(f, "stage_clocks")) return A.qM;   // [n][2 NM_MAX] reals, words 0.. the stage clocks of the last step sub-step (step_core.inl STAGE_CLOCK)
#endif
    return nullptr;
  }
  bool get_counters(int *out) override {
    CUDA_OK(cudaSetDevice(device));
    CUDA_OK(cudaMemcpyAsync(out, A.counters, sizeof(int) * n * 8, cudaMemcpyDeviceToHost, stream)); CUDA_OK(cudaStreamSynchronize(stream));
    return true;
  }
  int debug_dump(int env, double *out, int cnt) override {
    if (!A.dbg || env < 0 || env >= n) return -1;
    std::vector<real> t(D_SIZE);
    cudaSetDevice(device);
    if (cudaMemcpyAsync(t.data(), A.dbg + (size_t)env * D_SIZE, sizeof(real) * D_SIZE, cudaMemcpyDeviceToHost, stream) != cudaSuccess || cudaStreamSynchronize(stream) != cudaSuccess) return -1;
    if (cnt > D_SIZE) cnt = D_SIZE;
    for (int i = 0; i < cnt; i++) out[i] = (double)t[i];
    return cnt;
  }
};

}  // namespace cassie

// ====================================================================== C-ABI
using namespace cassie;
static_assert(CASSIE_CAM_MAXDIM == CAM_MAXDIM && CASSIE_CAM_MAX == CAM_MAX && CASSIE_CAMENV_SLOT == CAMENV_SLOT, "camera set and rows");
static_assert(CASSIE_RAY_MAX == RAY_MAX && CASSIE_RAY_SLOT == RAY_SLOT && CASSIE_RAY_HEADING == RAY_HEADING && CASSIE_RAY_ROOT == RAY_ROOT && CASSIE_RAY_WORLD == RAY_WORLD, "ray table and rows");
static_assert(CASSIE_FRAME_JAC_WIDTH == FRAME_JAC_W && CASSIE_FRAME_JAC_COLS == FJ_COLS, "frame Jacobian row layout");
static_assert(CASSIE_DYN_WIDTH == DYN_W && CASSIE_DYN_COLS == DY_COLS && CASSIE_DYN_M == DY_M && CASSIE_DYN_BIAS == DY_BIAS && CASSIE_DYN_JEQ == DY_JEQ && CASSIE_DYN_EQPOS == DY_EQPOS && CASSIE_DYN_RCM == DY_RCM, "dynamics row layout");
static_assert(CASSIE_INV_WIDTH == INV_W && CASSIE_INV_COLS == IV_COLS && CASSIE_INV_QFRC == IV_QFRC && CASSIE_INV_QFRCC == IV_QFRCC && CASSIE_INV_NEFC == IV_NEFC && CASSIE_INV_NCON == IV_NCON && CASSIE_INV_DROPPED == IV_DROPPED, "inverse row layout");
static_assert(CASSIE_ACC_QACC == AC_QACC && CASSIE_ACC_QCOLS == AC_QCOLS && CASSIE_ACC_CACC == AC_CACC && CASSIE_ACC_SLOT == AC_SLOT && CASSIE_ACC_WIDTH(3) == acc_width(3), "acceleration row layout");
static_assert(CASSIE_IK_MAX == IK_MAX && CASSIE_IK_TARGET_WIDTH == IK_TW && CASSIE_IK_SLOT == IK_SLOT && CASSIE_IK_MAX_ITER == IK_MAX_ITER && CASSIE_IK_WORLD == IK_WORLD && CASSIE_IK_ROOT == IK_ROOT &&
              CASSIE_IK_POS == IT_POS && CASSIE_IK_QUAT == IT_QUAT && CASSIE_IK_VEL == IT_VEL && CASSIE_IK_ANGVEL == IT_ANGVEL && CASSIE_IK_POS_RESIDUAL == IS_POS && CASSIE_IK_ORI_RESIDUAL == IS_ORI &&
              CASSIE_IK_LOOP_RESIDUAL == IS_LOOP && CASSIE_IK_ITERATIONS == IS_ITER && CASSIE_IK_OUTCOME == IS_OUTCOME && CASSIE_IK_JEQ_QVEL == IS_JV && CASSIE_IK_VEL_RESIDUAL == IS_VEL &&
              CASSIE_IK_AT_BOUND == IS_BOUND, "inverse-kinematics rows");
static_assert(CASSIE_LOOP_SLOT == LOOP_SLOT && CASSIE_LOOP_MAX_ITER == LOOP_MAX_ITER && CASSIE_LOOP_RESIDUAL == 0 && CASSIE_LOOP_ITERATIONS == 1 && CASSIE_LOOP_VEL_RESIDUAL == 2, "loop status rows");
static_assert(CASSIE_APPLIED_WIDTH == APPLIED_W && CASSIE_APPLIED_XFRC == AP_XFRC && CASSIE_APPLIED_QFRC == AP_QFRC, "applied-force row layout");
static_assert(CASSIE_SENSOR_WIDTH == SN_W && CASSIE_SN_ENC_OFF == SN_ENC_OFF && CASSIE_SN_ENC_STD == SN_ENC_STD && CASSIE_SN_QUAT == SN_QUAT && CASSIE_SN_ORI_STD == SN_ORI_STD && CASSIE_SN_GYRO_BIAS == SN_GYRO_BIAS && CASSIE_SN_GYRO_STD == SN_GYRO_STD && CASSIE_SN_ACC_BIAS == SN_ACC_BIAS && CASSIE_SN_ACC_STD == SN_ACC_STD, "sensor row layout");
static_assert(CASSIE_CON_WIDTH == CON_W && CASSIE_CON_MAX == MAXCON && CASSIE_CON_HEAD == CON_HEAD && CASSIE_CON_SLOT == CON_SLOT && CASSIE_CON_GEOM1 == CN_GEOM1 && CASSIE_CON_GEOM2 == CN_GEOM2 &&
              CASSIE_CON_DIM == CN_DIM && CASSIE_CON_DIST == CN_DIST && CASSIE_CON_POS == CN_POS && CASSIE_CON_FRAME == CN_FRAME && CASSIE_CON_FORCE == CN_FORCE && CASSIE_CON_MU == CN_MU &&
              CASSIE_CON_EFC == CN_EFC, "contact-list row layout");
static_assert(CASSIE_TRACE_QPOS == TC_QPOS && CASSIE_TRACE_QVEL == TC_QVEL && CASSIE_TRACE_OBS == TC_OBS && CASSIE_TRACE_AUX == TC_AUX && CASSIE_TRACE_FRAME == TC_FRAME && CASSIE_TRACE_MAX == TRACE_MAX, "trace sources");
static_assert(CASSIE_FRAME_WIDTH == FRAME_W && CASSIE_FRAME_POS == FR_POS && CASSIE_FRAME_QUAT == FR_QUAT && CASSIE_FRAME_VEL == FR_VEL && CASSIE_FRAME_CFRC == FR_CFRC && CASSIE_FRAME_MAX == FRAME_MAX, "frame row layout");
struct cassie_batch { BatchBase *impl; std::vector<double> obs, radio; };
struct cassie_sim { cassie_batch *b; double qpos[64], qvel[64], time, qpos_dev[64], qvel_dev[64], time_dev, aux[AUX_W]; std::vector<float> hfield, hfield_dev; std::string path; double timestep = 0, timestep_dev = 0;
  std::vector<double> m_mass, m_ipos, m_damp, m_fric, m_mass_dev, m_ipos_dev, m_damp_dev, m_fric_dev;
  std::vector<double> m_gpos, m_gquat, m_gsize, m_gpos_dev, m_gquat_dev, m_gsize_dev;
  // every body and every site is a frame of the simulator's batch (bodies first); host mirrors laid out like mjData's xpos[nbody][3], xquat[nbody][4],
  // site_xpos[nsite][3], so that the borrowed pointers of cassie_sim_xpos / xquat / site_xpos index across bodies as &d->xpos[3 * id] does
  std::vector<double> frames, xpos, xquat, site_xpos;
  // the acceleration row of the simulator's batch (qacc, then the cacc of every body and site frame) and the nv-entry qacc mirror cassie_sim_qacc lends out
  std::vector<double> acc, qacc;
  // the height field's size (cassie_sim_get_hfield_size / set_hfield_size): a host mirror, uploaded before the next launch when it is valid
  double hf_size[4] = {0, 0, 0, 0}, hf_size_dev[4] = {0, 0, 0, 0};
  // body offsets (cassie_sim_get_body_name_pos / set_body_name_pos): [nbody][3] host mirror; the constant block is rebuilt from it when it changes
  std::vector<double> m_bpos, m_bpos_dev;
  // the controller-stage state lent out by cassie_sim_joint_filter / drive_filter / ctrl: host mirrors laid out as joint_filter_t[6] (x[4], y[3]),
  // drive_filter_t[10] (int x[9]) and mjData's ctrl[nu].  Refreshed after every launch once one was lent; the filter mirrors are uploaded before the
  // next launch when they were written, ctrl is read-only in effect (the next step overwrites it, as cassie_motor_data does in the reference)
  double jfilt[6][7], jfilt_dev[6][7], ctrl[MU]; int dfilt[10][9], dfilt_dev[10][9]; bool act_lent = false, ctrl_zero = false;
  // qfrc_applied lent out by cassie_sim_qfrc: a host mirror of the batch's applied-force row [nv] (empty until the first call), uploaded before the next
  // launch when it was written, refreshed after every launch
  std::vector<double> qfrc, qfrc_dev; };   // geom placement (stair boxes): host mirrors, the constant block is rebuilt when they change   // host mirrors of the model arrays handed out as borrowed pointers

// cassie_state_t (include/cassiemujoco.h:434-463): a device-resident snapshot of one simulator's rows plus the host mirrors the reference hands out as
// borrowed pointers (time, qpos, qvel); the snapshot is allocated by the first cassie_get_state, which also fixes the owning simulator's sizes
struct cassie_state { cassie::Snap *snap = nullptr; double qpos[64], qvel[64], time = 0, qpos_snap[64], qvel_snap[64], time_snap = 0;
  bool ctrl_zero = false; };   // the simulator's ctrl read zeros when the snapshot was taken (after cassie_sim_full_reset, before a step)

static std::mutex g_model_mutex;
static std::string g_model_path;   // what cassie_mujoco_init cached (the reference caches the parsed model, src/cassiemujoco.c:48-59)

// the name table of an object kind (mj_name2id's type strings), or null with a recorded error: the compiled model keeps the names of bodies (also as
// "xbody", as MuJoCo does), joints, geoms, sites and cameras; mj_name2id's other kinds have no table here, and an unknown kind is MuJoCo's mjOBJ_UNKNOWN
static const std::vector<std::string> *name_table(const HostModel &m, const char *type, const char *verb) {
  const std::string t = type ? type : "";
  if (t == "body" || t == "xbody") return &m.names_body;
  if (t == "joint") return &m.names_joint;
  if (t == "geom") return &m.names_geom;
  if (t == "site") return &m.names_site;
  if (t == "camera") return &m.names_camera;
  static const char *const others[] = {"dof", "light", "mesh", "skin", "hfield", "texture", "material", "pair", "exclude", "equality", "tendon", "actuator",
                                       "sensor", "numeric", "text", "tuple", "key"};
  for (const char *o : others) if (t == o) { set_err(std::string(verb) + ": the compiled model keeps no names of kind " + t); return nullptr; }
  set_err(std::string(verb) + ": unknown object type " + (type ? "\"" + t + "\"" : std::string("(null)")));
  return nullptr;
}

extern "C" {

const char *cassie_b200_last_error(void) { return g_err.c_str(); }

cassie_batch_t *cassie_batch_init(const char *modelfile, int n_env, int device, int precision) {
  g_err.clear();
  if (!modelfile || n_env <= 0) { set_err("cassie_batch_init: bad arguments"); return nullptr; }
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) { set_err("no CUDA device: the batched stepper has no CPU fallback"); return nullptr; }
  if (device < 0 || device >= ndev) { set_err("bad device index"); return nullptr; }
  BatchBase *impl = precision == CASSIE_B200_FP64 ? (BatchBase *)new Batch<double>() : (BatchBase *)new Batch<float>();
  std::string err;
  if (!load_model_any(modelfile, impl->hm, err)) { set_err("Load model error: " + err); delete impl; return nullptr; }
  impl->n = n_env; impl->device = device; impl->precision = precision; impl->debug = getenv("CASSIE_B200_DEBUG") != nullptr;
  if (!impl->init() || !impl->sync()) { delete impl; return nullptr; }
  cassie_batch *b = new cassie_batch(); b->impl = impl; b->radio.assign((size_t)n_env * 16, 0.0);
  for (int e = 0; e < n_env; e++) b->radio[(size_t)e * 16 + 8] = 1.0;
  return b;
}
void cassie_batch_free(cassie_batch_t *b) { if (!b) return; delete b->impl; delete b; }
int cassie_batch_nenv(const cassie_batch_t *b) { return b->impl->n; }
int cassie_batch_nq(const cassie_batch_t *b) { return b->impl->hm.nq; }
int cassie_batch_nv(const cassie_batch_t *b) { return b->impl->hm.nv; }
int cassie_batch_precision(const cassie_batch_t *b) { return b->impl->precision; }
int cassie_batch_row_width(const cassie_batch_t *b, const char *field) {
  if (!strcmp(field, "qpos")) return b->impl->hm.nq > 36 ? QPOS_W_XB : QPOS_W_MAIN; if (!strcmp(field, "qvel")) return b->impl->hm.nv > 32 ? QVEL_W_XB : QVEL_W_MAIN;
  if (!strcmp(field, "pd")) return PD_W; if (!strcmp(field, "obs")) return OBS_W; if (!strcmp(field, "xfrc")) return XFRC_W; if (!strcmp(field, "aux")) return AUX_W;
  if (!strcmp(field, "frames")) return (int)(b->impl->frame_list.size() / 2) * FRAME_W; if (!strcmp(field, "frame_jac")) return FRAME_JAC_W;
  if (!strcmp(field, "dyn")) return DYN_W; if (!strcmp(field, "rays")) return b->impl->nray * RAY_SLOT;
  if (!strcmp(field, "depth") || !strcmp(field, "camera_geom")) return b->impl->cam.k * b->impl->cam.width * b->impl->cam.height; if (!strcmp(field, "camera_env")) return b->impl->cam.k * CAMENV_SLOT; if (!strcmp(field, "terrain")) return 1; if (!strcmp(field, "actuators")) return ACT_W; if (!strcmp(field, "mechanics")) return MECH_W; if (!strcmp(field, "contact")) return CONTACT_W; if (!strcmp(field, "applied")) return APPLIED_W;
  if (!strcmp(field, "trace")) return b->impl->trace_width();
  if (!strcmp(field, "contacts")) return CON_W; if (!strcmp(field, "loops")) return LOOP_SLOT; if (!strcmp(field, "ik_targets")) return IK_MAX * IK_TW; if (!strcmp(field, "ik")) return IK_SLOT;
  if (!strcmp(field, "sensors")) return SN_W; if (!strcmp(field, "sensor_rng")) return SR_W;
  if (!strcmp(field, "inv_qacc")) return b->impl->hm.nv > 32 ? QVEL_W_XB : QVEL_W_MAIN; if (!strcmp(field, "inv")) return INV_W;
  if (!strcmp(field, "acc")) return acc_width((int)(b->impl->frame_list.size() / 2)); return -1;
}
long cassie_batch_launch_count(const cassie_batch_t *b) { return b->impl->launches; }
void cassie_batch_reset(cassie_batch_t *b, const unsigned char *mask) { b->impl->reset(mask); b->impl->sync(); b->impl->reset_estimator(mask); b->impl->reset_estimator_device(mask); }   // a fresh cassie_sim_t has a fresh estimator
void cassie_batch_set_pd(cassie_batch_t *b, const double *pd) { b->impl->set_pd(pd); }
void cassie_batch_step(cassie_batch_t *b, int nticks) { if (nticks > 0) b->impl->step(nticks, 0); }
void cassie_batch_forward(cassie_batch_t *b) { b->impl->step(0, 1); }
void cassie_batch_sync(cassie_batch_t *b) { b->impl->sync(); }
void cassie_batch_get_qpos(cassie_batch_t *b, double *out) { b->impl->get("qpos", out); }
void cassie_batch_set_qpos(cassie_batch_t *b, const double *in) { b->impl->set("qpos", in); }
void cassie_batch_get_qvel(cassie_batch_t *b, double *out) { b->impl->get("qvel", out); }
void cassie_batch_set_qvel(cassie_batch_t *b, const double *in) { b->impl->set("qvel", in); }
void cassie_batch_get_time(cassie_batch_t *b, double *out) { b->impl->get("time", out); }
void cassie_batch_get_obs(cassie_batch_t *b, double *out) { b->impl->get("obs", out); }
int cassie_batch_nbody(const cassie_batch_t *b) { return b->impl->hm.nbody; }
int cassie_batch_ngeom(const cassie_batch_t *b) { return b->impl->hm.ngeom; }
int cassie_batch_njnt(const cassie_batch_t *b) { return b->impl->hm.njnt; }
int cassie_batch_set_body_mass(cassie_batch_t *b, const double *mass) { return b->impl->set_model_rows("body_mass", mass, b->impl->hm.nbody) ? 0 : -1; }
int cassie_batch_set_body_ipos(cassie_batch_t *b, const double *ipos) { return b->impl->set_model_rows("body_ipos", ipos, 3 * b->impl->hm.nbody) ? 0 : -1; }
int cassie_batch_set_dof_damping(cassie_batch_t *b, const double *damp) { return b->impl->set_model_rows("dof_damping", damp, b->impl->hm.nv) ? 0 : -1; }
int cassie_batch_set_geom_friction(cassie_batch_t *b, const double *fric) { return b->impl->set_model_rows("geom_friction", fric, 3 * b->impl->hm.ngeom) ? 0 : -1; }
int cassie_batch_get_body_mass(cassie_batch_t *b, double *mass) { return b->impl->get_model_rows("body_mass", mass, b->impl->hm.nbody) ? 0 : -1; }
int cassie_batch_get_body_ipos(cassie_batch_t *b, double *ipos) { return b->impl->get_model_rows("body_ipos", ipos, 3 * b->impl->hm.nbody) ? 0 : -1; }
int cassie_batch_get_dof_damping(cassie_batch_t *b, double *damp) { return b->impl->get_model_rows("dof_damping", damp, b->impl->hm.nv) ? 0 : -1; }
int cassie_batch_get_geom_friction(cassie_batch_t *b, double *fric) { return b->impl->get_model_rows("geom_friction", fric, 3 * b->impl->hm.ngeom) ? 0 : -1; }
int cassie_batch_set_const(cassie_batch_t *b, const unsigned char *mask, int reset_state) { return b->impl->set_const(mask, reset_state != 0) ? 0 : -1; }
int cassie_batch_set_task_pd(cassie_batch_t *b, const double *rows) { return b->impl->set_task_pd(rows) ? 0 : -1; }
int cassie_batch_set_pd_gait(cassie_batch_t *b, const double *amp, const double *freq, const double *phase) { return b->impl->set_pd_gait(amp, freq, phase) ? 0 : -1; }
int cassie_batch_enable_estimator_forces(cassie_batch_t *b, int on) { b->impl->est_forces = on != 0; return 0; }
void cassie_b200_estimator_leg_force(int side, const double ang[7], const double quat[4], double force[3]) { estimator_leg_force(side, ang, quat, force); }
int cassie_batch_enable_estimator_filter(cassie_batch_t *b, int on) { b->impl->est_filter = on != 0; if (on) b->impl->est_forces = true; else b->impl->est_state.clear(); return 0; }
int cassie_batch_reset_estimator(cassie_batch_t *b, const unsigned char *mask) { b->impl->reset_estimator(mask); return b->impl->reset_estimator_device(mask) ? 0 : -1; }
// the same filters as a plain host object (no GPU involved): what the unpack loop above runs per environment
void *cassie_b200_estimator_filter_new(void) { return new cassie::EstimatorFilter(); }
void cassie_b200_estimator_filter_free(void *f) { delete static_cast<cassie::EstimatorFilter *>(f); }
void cassie_b200_estimator_filter_reset(void *f) { static_cast<cassie::EstimatorFilter *>(f)->reset(); }
void cassie_b200_estimator_filter_step(void *f, state_out_t *y) {
  static_cast<cassie::EstimatorFilter *>(f)->step(y->pelvis.orientation, y->leftFoot.position, y->rightFoot.position, y->leftFoot.toeForce[2] + y->leftFoot.heelForce[2],
      y->rightFoot.toeForce[2] + y->rightFoot.heelForce[2], y->pelvis.translationalAcceleration, y->pelvis.position, y->pelvis.translationalVelocity, y->pelvis.externalForce, &y->terrain.height);
}
int cassie_batch_enable_aux(cassie_batch_t *b, int on) { return b->impl->enable_aux(on != 0) ? 0 : -1; }
int cassie_batch_get_aux(cassie_batch_t *b, double *out) { return b->impl->get("aux", out) ? 0 : -1; }
int cassie_batch_enable_estimator_device(cassie_batch_t *b, int on) { if (!on) b->impl->est_auto = false; return b->impl->enable_estimator_device(on != 0) ? 0 : -1; }
int cassie_batch_get_estimator(cassie_batch_t *b, double *out) { return b->impl->get("est_out", out) ? 0 : -1; }
int cassie_batch_query(cassie_batch_t *b) { if (!b->impl->has_aux() && !b->impl->enable_aux(true)) return -1; return b->impl->step(0, 2) ? 0 : -1; }
int cassie_batch_apply_force(cassie_batch_t *b, const double *xfrc, const char *body_name) {
  int id = body_name ? b->impl->hm.body_id(body_name) : -1;
  if (id <= 0) { set_err("cassie_batch_apply_force: unknown body (no-op)"); return -1; }
  return b->impl->set_xfrc(xfrc, id) ? 0 : -1;
}
void cassie_batch_clear_forces(cassie_batch_t *b) { b->impl->set_xfrc(nullptr, 0); b->impl->clear_applied_xfrc(); }
void cassie_batch_integrate_pos(cassie_batch_t *b) { b->impl->integrate(); }
int cassie_batch_set_hfielddata(cassie_batch_t *b, const float *data, int n_terrains) { return b->impl->set_hfield(data, n_terrains) ? 0 : -1; }
int cassie_batch_hfield_nrow(const cassie_batch_t *b) { return b->impl->hm.nhfield ? b->impl->hm.hfield_nrow[0] : 0; }
int cassie_batch_hfield_ncol(const cassie_batch_t *b) { return b->impl->hm.nhfield ? b->impl->hm.hfield_ncol[0] : 0; }
void *cassie_batch_device_ptr(cassie_batch_t *b, const char *field) { return b->impl->dev_ptr(field); }
void cassie_batch_set_stream(cassie_batch_t *b, void *s) { b->impl->sync(); if (b->impl->own_stream && b->impl->stream) cudaStreamDestroy(b->impl->stream); b->impl->stream = (cudaStream_t)s; b->impl->own_stream = false; }
void *cassie_batch_get_stream(cassie_batch_t *b) { return (void *)b->impl->stream; }
void cassie_batch_get_counters(cassie_batch_t *b, int *out) { b->impl->get_counters(out); }
int cassie_batch_debug_dump(cassie_batch_t *b, int env, double *out, int n) { return b->impl->debug_dump(env, out, n); }

void cassie_batch_aos_timing(cassie_batch_t *b, double out[6], int reset) { for (int i = 0; i < 6; i++) out[i] = b->impl->aos_t[i]; if (reset) for (int i = 0; i < 6; i++) b->impl->aos_t[i] = 0; }
int cassie_b200_aos_threads(void) { return cassie::aos_thread_count(); }
int cassie_b200_effective_cpus(void) { return cassie::effective_cpus(); }
void cassie_sim_step_pd_batch(cassie_batch_t *b, const pd_in_t *pd_in, state_out_t *state_out) {
  b->impl->step_pd_aos(pd_in, state_out, b->radio.data());
}

// ---------------- legacy single-environment verbs
bool cassie_mujoco_init(const char *modelfile) {
  std::lock_guard<std::mutex> g(g_model_mutex);
  if (!g_model_path.empty()) return true;
  if (!modelfile) { set_err("cassie_mujoco_init: model file required"); return false; }
  HostModel hm; std::string err;
  if (!load_model_any(modelfile, hm, err)) { fprintf(stderr, "Load model error: %s\n", err.c_str()); g_err = err; return false; }
  g_model_path = modelfile; return true;
}
void cassie_cleanup(void) { std::lock_guard<std::mutex> g(g_model_mutex); g_model_path.clear(); }
static void sim_pull_act(cassie_sim_t *c) {   // the controller-stage mirrors, once lent out; a filter mirror written and not yet uploaded is kept
  double cst[CST_W]; int df[90];   // one download of the controller row (joint filters, drive torques) and one of the FIR taps
  if (!c->b->impl->get("cst", cst) || !c->b->impl->get_actuator_state(nullptr, df, nullptr, nullptr)) return;
  if (!memcmp(c->jfilt, c->jfilt_dev, sizeof c->jfilt)) {
    for (int j = 0; j < 6; j++) { for (int k = 0; k < 4; k++) c->jfilt[j][k] = cst[CS_JFX + 4 * j + k]; for (int k = 0; k < 3; k++) c->jfilt[j][4 + k] = cst[CS_JFY + 3 * j + k]; }
    memcpy(c->jfilt_dev, c->jfilt, sizeof c->jfilt); }
  if (!memcmp(c->dfilt, c->dfilt_dev, sizeof c->dfilt)) { memcpy(c->dfilt, df, sizeof c->dfilt); memcpy(c->dfilt_dev, c->dfilt, sizeof c->dfilt); }
  const HostModel &hm = c->b->impl->hm;   // the ctrl the last physics step applied: the drive torque over the gear (src/cassiemujoco.c:660-662)
  for (int i = 0; i < hm.nu && i < MU; i++) c->ctrl[i] = c->ctrl_zero ? 0.0 : cst[CS_DTORQUE + i] / hm.actuator_gear[i];
}
static void sim_pull(cassie_sim_t *c) {
  c->b->impl->get("qpos", c->qpos); c->b->impl->get("qvel", c->qvel); c->b->impl->get("time", &c->time); if (c->b->impl->has_aux()) c->b->impl->get("aux", c->aux);
  if (!c->frames.empty() && c->b->impl->get("frames", c->frames.data())) {   // the sizes were fixed at init: the borrowed pointers stay valid
    const int nb = (int)c->xquat.size() / 4, ns = (int)c->site_xpos.size() / 3;
    for (int b = 0; b < nb; b++) { const double *f = &c->frames[(size_t)b * FRAME_W]; for (int k = 0; k < 3; k++) c->xpos[3 * b + k] = f[FR_POS + k]; for (int k = 0; k < 4; k++) c->xquat[4 * b + k] = f[FR_QUAT + k]; }
    for (int s = 0; s < ns; s++) for (int k = 0; k < 3; k++) c->site_xpos[3 * s + k] = c->frames[(size_t)(nb + s) * FRAME_W + FR_POS + k];
  }
  if (!c->acc.empty() && c->b->impl->get("acc", c->acc.data())) for (int i = 0; i < c->b->impl->hm.nv; i++) c->qacc[i] = c->acc[AC_QACC + i];
  memcpy(c->qpos_dev, c->qpos, sizeof c->qpos); memcpy(c->qvel_dev, c->qvel, sizeof c->qvel); c->time_dev = c->time;
  if (c->act_lent) sim_pull_act(c);
  if (!c->qfrc.empty() && c->b->impl->get_applied_forces(nullptr, c->qfrc.data())) c->qfrc_dev = c->qfrc;
}
static void sim_lend_act(cassie_sim_t *c) { if (!c->act_lent) { c->act_lent = true; sim_pull_act(c); } }   // the first lend fills the mirrors
static void sim_push(cassie_sim_t *c) {  // upload whatever the caller wrote through the borrowed pointers
  if (memcmp(c->qpos_dev, c->qpos, sizeof c->qpos)) c->b->impl->set("qpos", c->qpos);
  if (memcmp(c->qvel_dev, c->qvel, sizeof c->qvel)) c->b->impl->set("qvel", c->qvel);
  if (c->time_dev != c->time) c->b->impl->set("time", &c->time);
  if (c->timestep != c->timestep_dev) { if (c->timestep > 0) { c->b->impl->hm.timestep = c->timestep; c->b->impl->rebuild_model(); } c->timestep_dev = c->timestep; }   // written through cassie_sim_timestep()
  if (!c->hfield.empty() && c->hfield != c->hfield_dev) { c->b->impl->set_hfield(c->hfield.data(), 1); c->hfield_dev = c->hfield; }
  if (c->b->impl->hm.nhfield && memcmp(c->hf_size, c->hf_size_dev, sizeof c->hf_size)) {   // an invalid size is not uploaded: the error is recorded once, the last valid size stays
    cassie_batch_set_hfield_size(c->b, c->hf_size); memcpy(c->hf_size_dev, c->hf_size, sizeof c->hf_size); }
  if (c->m_mass != c->m_mass_dev) { cassie_batch_set_body_mass(c->b, c->m_mass.data()); c->m_mass_dev = c->m_mass; }
  if (c->m_ipos != c->m_ipos_dev) { cassie_batch_set_body_ipos(c->b, c->m_ipos.data()); c->m_ipos_dev = c->m_ipos; }
  if (c->m_damp != c->m_damp_dev) { cassie_batch_set_dof_damping(c->b, c->m_damp.data()); c->m_damp_dev = c->m_damp; }
  if (c->m_fric != c->m_fric_dev) { cassie_batch_set_geom_friction(c->b, c->m_fric.data()); c->m_fric_dev = c->m_fric; }
  if (c->m_gpos != c->m_gpos_dev || c->m_gquat != c->m_gquat_dev || c->m_gsize != c->m_gsize_dev) {   // a geom was moved / turned / resized (src/cassiemujoco.c:1438-1541)
    HostModel &hm = c->b->impl->hm; hm.geom_pos = c->m_gpos; hm.geom_quat = c->m_gquat; hm.geom_size = c->m_gsize;
    c->b->impl->rebuild_model(); c->m_gpos_dev = c->m_gpos; c->m_gquat_dev = c->m_gquat; c->m_gsize_dev = c->m_gsize; }
  if (c->m_bpos != c->m_bpos_dev) {   // a body was moved (src/cassiemujoco.c:1408-1418): kinematics, static geoms' world poses and the broad phase's bound follow
    c->b->impl->hm.body_pos = c->m_bpos; c->b->impl->rebuild_model(); c->m_bpos_dev = c->m_bpos; }
  if (c->act_lent && memcmp(c->jfilt, c->jfilt_dev, sizeof c->jfilt)) {   // written through cassie_sim_joint_filter (src/cassiemujoco.c:2119-2121)
    double jx[24], jy[18];
    for (int j = 0; j < 6; j++) { for (int k = 0; k < 4; k++) jx[4 * j + k] = c->jfilt[j][k]; for (int k = 0; k < 3; k++) jy[3 * j + k] = c->jfilt[j][4 + k]; }
    c->b->impl->set_actuator_state(nullptr, nullptr, jx, jy, nullptr); memcpy(c->jfilt_dev, c->jfilt, sizeof c->jfilt); }
  if (c->act_lent && memcmp(c->dfilt, c->dfilt_dev, sizeof c->dfilt)) {   // written through cassie_sim_drive_filter (:2151-2153)
    c->b->impl->set_actuator_state(nullptr, &c->dfilt[0][0], nullptr, nullptr, nullptr); memcpy(c->dfilt_dev, c->dfilt, sizeof c->dfilt); }
  if (c->qfrc != c->qfrc_dev && c->b->impl->set_applied_forces(nullptr, c->qfrc.data(), nullptr)) c->qfrc_dev = c->qfrc;   // written through cassie_sim_qfrc
}
cassie_sim_t *cassie_sim_init(const char *modelfile, bool reinit) {
  std::string path;
  { std::lock_guard<std::mutex> g(g_model_mutex); if (reinit || g_model_path.empty()) { if (!modelfile) { set_err("cassie_sim_init: model file required"); return nullptr; } path = modelfile; if (g_model_path.empty()) g_model_path = modelfile; } else path = g_model_path; }
  cassie_batch_t *b = cassie_batch_init(path.c_str(), 1, 0, CASSIE_B200_FP64);
  if (!b) return nullptr;
  cassie_sim_t *c = new cassie_sim(); memset(c->qpos, 0, sizeof c->qpos); memset(c->qvel, 0, sizeof c->qvel); memset(c->aux, 0, sizeof c->aux); c->b = b; c->path = path; c->timestep = c->timestep_dev = b->impl->hm.timestep;
  b->impl->legacy = true;
  b->impl->enable_aux(true);   // a single environment always carries the derived-quantity row ...
  { const HostModel &hm = b->impl->hm; std::vector<const char *> names; std::vector<int> kinds;   // ... and a frame per body and site (cassie_sim_xpos & co.)
    for (const std::string &s : hm.names_body) { names.push_back(s.c_str()); kinds.push_back(0); }
    for (const std::string &s : hm.names_site) { names.push_back(s.c_str()); kinds.push_back(1); }
    if ((int)names.size() <= FRAME_MAX && (int)hm.names_body.size() == hm.nbody && b->impl->set_frames(names.data(), kinds.data(), (int)names.size())) {
      c->frames.assign(names.size() * FRAME_W, 0.0); c->xpos.assign(3 * hm.names_body.size(), 0.0); c->xquat.assign(4 * hm.names_body.size(), 0.0); c->site_xpos.assign(3 * hm.names_site.size(), 0.0); } }
  c->qacc.assign(64, 0.0);   // ... and the acceleration row (cassie_sim_qacc, cassie_sim_body_acceleration)
  if (b->impl->enable_accelerations(true)) c->acc.assign(acc_width((int)(c->frames.size() / FRAME_W)), 0.0);
  b->impl->step(0, 1);   // populate them like the sensordata
  b->impl->enable_estimator_device(true);   // ... and the estimator (toe / heel forces, filters) inside the kernel, as state_output_step runs in every cassie_sim_step_pd (src/cassiemujoco.c:1156)
  sim_pull(c);
  { const HostModel &hm = b->impl->hm; c->m_mass = hm.body_mass; c->m_ipos = hm.body_ipos; c->m_damp = hm.dof_damping; c->m_fric = hm.geom_friction;
    c->m_mass_dev = c->m_mass; c->m_ipos_dev = c->m_ipos; c->m_damp_dev = c->m_damp; c->m_fric_dev = c->m_fric;
    c->m_gpos = hm.geom_pos; c->m_gquat = hm.geom_quat; c->m_gsize = hm.geom_size; c->m_gpos_dev = c->m_gpos; c->m_gquat_dev = c->m_gquat; c->m_gsize_dev = c->m_gsize;
    c->m_bpos = c->m_bpos_dev = hm.body_pos; }
  if (b->impl->hm.nhfield) { c->hfield.assign((size_t)b->impl->hm.hfield_nrow[0] * b->impl->hm.hfield_ncol[0], 0.0f); c->hfield_dev = c->hfield;
                             for (int k = 0; k < 4; k++) c->hf_size[k] = c->hf_size_dev[k] = b->impl->hm.hfield_size[k]; }
  return c;
}
// the one-environment batch a simulator steps: batch verbs (per-environment rows, device pointers) apply to it; owned by the simulator
cassie_batch_t *cassie_sim_batch(cassie_sim_t *c) { return c ? c->b : nullptr; }
void cassie_sim_free(cassie_sim_t *c) { if (!c) return; cassie_batch_free(c->b); delete c; }
void cassie_sim_step_pd(cassie_sim_t *c, state_out_t *y, const pd_in_t *u) { sim_push(c); cassie_sim_step_pd_batch(c->b, u, y); c->ctrl_zero = false; sim_pull(c); }
double *cassie_sim_time(cassie_sim_t *c) { return &c->time; }
double *cassie_sim_qpos(cassie_sim_t *c) { return c->qpos; }
double *cassie_sim_qvel(cassie_sim_t *c) { return c->qvel; }
// :1232-1235: mjData's qfrc_applied [nv] as a borrowed host mirror, uploaded before the next launch like qpos; the first call gives the simulator's batch
// its applied-force rows
double *cassie_sim_qfrc(cassie_sim_t *c) {
  if (c->qfrc.empty()) {
    if (!c->b->impl->enable_applied_forces(true)) return nullptr;
    c->qfrc.assign(c->b->impl->hm.nv, 0.0);
    if (!c->b->impl->get_applied_forces(nullptr, c->qfrc.data())) return nullptr;
    c->qfrc_dev = c->qfrc;
  }
  return c->qfrc.data();
}
int cassie_sim_nv(const cassie_sim_t *c) { return c->b->impl->hm.nv; }
int cassie_sim_nq(const cassie_sim_t *c) { return c->b->impl->hm.nq; }
void cassie_sim_apply_force(cassie_sim_t *c, double xfrc[6], const char *name) { cassie_batch_apply_force(c->b, xfrc, name); }
void cassie_sim_clear_forces(cassie_sim_t *c) { cassie_batch_clear_forces(c->b); }
void cassie_sim_radio(cassie_sim_t *c, double channels[16]) { for (int i = 0; i < 16; i++) c->b->radio[i] = channels[i]; double s = channels[8]; c->b->impl->set("sto", &s); }
int cassie_sim_get_hfield_nrow(cassie_sim_t *c) { return cassie_batch_hfield_nrow(c->b); }
int cassie_sim_get_hfield_ncol(cassie_sim_t *c) { return cassie_batch_hfield_ncol(c->b); }
int cassie_sim_get_nhfielddata(cassie_sim_t *c) { return (int)c->hfield.size(); }
float *cassie_sim_hfielddata(cassie_sim_t *c) { return c->hfield.empty() ? nullptr : c->hfield.data(); }
void cassie_sim_set_hfielddata(cassie_sim_t *c, float *data) { for (size_t i = 0; i < c->hfield.size(); i++) c->hfield[i] = data[i]; }
// src/cassiemujoco.c:2062-2070: a borrowed pointer to the height field's size [x half-extent, y half-extent, elevation scale, base thickness], uploaded
// before the next step or forward like the elevations
double *cassie_sim_get_hfield_size(cassie_sim_t *c) {
  if (!c->b->impl->hm.nhfield) { set_err("cassie_sim_get_hfield_size: this model has no height field"); return nullptr; }
  return c->hf_size;
}
void cassie_sim_set_hfield_size(cassie_sim_t *c, double size[4]) {
  if (!c->b->impl->hm.nhfield) { set_err("cassie_sim_set_hfield_size: this model has no height field"); return; }
  if (size) for (int k = 0; k < 4; k++) c->hf_size[k] = size[k];
}
// ---- read-only derived quantities (include/cassiemujoco.h:200-240).  Contact forces, flags, foot positions / velocities are by-products of
// the last step (the reference reads the same stale mjData arrays); the centre-of-mass group recomputes the kinematics of the CURRENT
// state first, as the reference does with mj_fwdPosition, through a query launch that writes nothing else.
static const double *sim_aux(const cassie_sim_t *c) { return c->aux; }
static void sim_query(const cassie_sim_t *cc) { cassie_sim_t *c = const_cast<cassie_sim_t *>(cc); sim_push(c); double keep[AUX_W]; memcpy(keep, c->aux, sizeof keep);
  cassie_batch_query(c->b); c->b->impl->get("aux", c->aux);
  for (int i = 0; i < AUX_W; i++) if (i < AX_CM_POS || i >= AX_ANGMOM + 3) c->aux[i] = keep[i]; }
void cassie_sim_foot_forces(const cassie_sim_t *c, double cfrc[12]) { memcpy(cfrc, sim_aux(c) + AX_FOOT_FORCE, 12 * sizeof(double)); }
void cassie_sim_heeltoe_forces(const cassie_sim_t *c, double toe_force[6], double heel_force[6]) { memcpy(toe_force, sim_aux(c) + AX_TOE_FORCE, 6 * sizeof(double)); memcpy(heel_force, sim_aux(c) + AX_HEEL_FORCE, 6 * sizeof(double)); }
void cassie_sim_foot_positions(const cassie_sim_t *c, double cpos[6]) { memcpy(cpos, sim_aux(c) + AX_FOOT_POS, 6 * sizeof(double)); }
void cassie_sim_foot_velocities(const cassie_sim_t *c, double cvel[12]) { memcpy(cvel, sim_aux(c) + AX_FOOT_VEL, 12 * sizeof(double)); }
void cassie_sim_cm_position(const cassie_sim_t *c, double cm_pos[3]) { sim_query(c); memcpy(cm_pos, sim_aux(c) + AX_CM_POS, 3 * sizeof(double)); }
void cassie_sim_cm_velocity(const cassie_sim_t *c, double cm_vel[3]) { sim_query(c); memcpy(cm_vel, sim_aux(c) + AX_CM_VEL, 3 * sizeof(double)); }
void cassie_sim_angular_momentum(const cassie_sim_t *c, double Lcm[3]) { sim_query(c); memcpy(Lcm, sim_aux(c) + AX_ANGMOM, 3 * sizeof(double)); }
bool cassie_sim_check_obstacle_collision(const cassie_sim_t *c) { return sim_aux(c)[AX_OBSTACLE] != 0; }
bool cassie_sim_check_self_collision(const cassie_sim_t *c) { return sim_aux(c)[AX_SELF] != 0; }
bool cassie_sim_geom_collision(const cassie_sim_t *c, int geom_group) { return geom_group >= 0 && geom_group < 16 && (((int)sim_aux(c)[AX_GROUPMASK] >> geom_group) & 1); }
// ---- frames (src/cassiemujoco.c:1242-1301, 1543-1562, 1752-1809): poses, cvel and contact forces are the frame rows the last step / forward left
// behind, kept in the simulator's mirrors; the Jacobians recompute the kinematics of the CURRENT state in a launch that writes nothing else (the
// reference's mj_kinematics there also overwrites d->xpos; the mirrors keep the last step's poses, as cassie_sim_cm_position leaves them).  An unknown
// name returns NULL / zeros and records an error (the reference indexes its arrays with -1).
static int sim_body(const cassie_sim_t *c, const char *name, const char *verb) {
  const int id = name && !c->frames.empty() ? c->b->impl->hm.body_id(name) : -1;
  if (id < 0) set_err(std::string(verb) + ": unknown body " + (name ? name : "(null)"));
  return id;
}
static int sim_site(const cassie_sim_t *c, const char *name, const char *verb) {
  const int id = name && !c->frames.empty() ? c->b->impl->hm.site_id(name) : -1;
  if (id < 0) set_err(std::string(verb) + ": unknown site " + (name ? name : "(null)"));
  return id;
}
static const double *sim_frame(const cassie_sim_t *c, int f) { return &c->frames[(size_t)f * FRAME_W]; }
double *cassie_sim_xpos(cassie_sim_t *c, const char *name) { const int b = sim_body(c, name, "cassie_sim_xpos"); return b < 0 ? nullptr : &c->xpos[3 * b]; }
double *cassie_sim_xquat(cassie_sim_t *c, const char *name) { const int b = sim_body(c, name, "cassie_sim_xquat"); return b < 0 ? nullptr : &c->xquat[4 * b]; }
double *cassie_sim_site_xpos(cassie_sim_t *c, const char *name) { const int s = sim_site(c, name, "cassie_sim_site_xpos"); return s < 0 ? nullptr : &c->site_xpos[3 * s]; }
void cassie_sim_site_xquat(cassie_sim_t *c, const char *name, double *xquat) {
  const int s = sim_site(c, name, "cassie_sim_site_xquat");
  for (int k = 0; k < 4; k++) xquat[k] = s < 0 ? 0.0 : sim_frame(c, (int)c->xquat.size() / 4 + s)[FR_QUAT + k];
}
// the six rangefinders (src/cassiemujoco.c:776-778, sensordata[29..35)): each site's ray along its z axis from the mirrors' site poses (those of the state
// the last sub-step started from, when MuJoCo evaluates mj_sensorPos), one world-frame cast on the simulator's batch of one, then MuJoCo's cutoff for a
// positive-type sensor: min(cutoff, d) where cutoff > 0 (a miss, -1, stays -1); no noise, as in the reference.  Slots without a rangefinder read 0.
// The rays see the static geoms only (DESIGN.md section 3).  A model without rangefinders gets zeros and a recorded error.
void cassie_sim_read_rangefinder(cassie_sim_t *c, double ranges[6]) {
  for (int i = 0; i < 6; i++) ranges[i] = 0;
  const HostModel &hm = c->b->impl->hm; const int k = std::min((int)hm.rangefinder_site.size(), 6), nb = (int)c->xquat.size() / 4;
  if (!k || c->frames.empty()) { set_err("cassie_sim_read_rangefinder: the model has no rangefinders"); return; }
  int kind[6]; double org[18], dir[18], maxd[6], out[6 * RAY_SLOT];
  for (int i = 0; i < k; i++) {
    const double *f = sim_frame(c, nb + hm.rangefinder_site[i]), *q = f + FR_QUAT;
    kind[i] = RAY_WORLD; maxd[i] = 1e6;   // mj_ray has no range limit
    for (int j = 0; j < 3; j++) org[3 * i + j] = f[FR_POS + j];
    dir[3 * i] = 2 * (q[1] * q[3] + q[0] * q[2]); dir[3 * i + 1] = 2 * (q[2] * q[3] - q[0] * q[1]); dir[3 * i + 2] = q[0] * q[0] - q[1] * q[1] - q[2] * q[2] + q[3] * q[3];
  }
  if (!c->b->impl->set_rays(kind, org, dir, maxd, k) || !c->b->impl->raycast() || !c->b->impl->get_rays(out)) return;
  for (int i = 0; i < k; i++) { const double d = out[RAY_SLOT * i], cut = hm.rangefinder_cutoff[i]; ranges[i] = (cut > 0 && d >= 0) ? std::min(cut, d) : d; }
}
void cassie_sim_body_velocities(const cassie_sim_t *c, double cvel[6], const char *name) {
  const int b = sim_body(c, name, "cassie_sim_body_velocities");
  for (int k = 0; k < 6; k++) cvel[k] = b < 0 ? 0.0 : sim_frame(c, b)[FR_VEL + k];
}
// ---- accelerations (src/cassiemujoco.c:1216-1219, 1762-1779): the acceleration row the last step / forward left behind, like the velocities above.  The
// reference reruns mj_comVel + mj_rnePostConstraint on mjData at call time; the two differ only when qvel was written through the borrowed pointer since.
double *cassie_sim_qacc(cassie_sim_t *c) { return c->qacc.data(); }
void cassie_sim_body_acceleration(const cassie_sim_t *c, double accel[6], const char *name) {
  const int b = sim_body(c, name, "cassie_sim_body_acceleration");
  for (int k = 0; k < 6; k++) accel[k] = (b < 0 || c->acc.empty()) ? 0.0 : c->acc[AC_CACC + AC_SLOT * b + k];
}
void cassie_sim_foot_orient(const cassie_sim_t *c, double corient[4]) {
  const int s = sim_site(c, "right-foot-middle", "cassie_sim_foot_orient");
  for (int k = 0; k < 4; k++) corient[k] = s < 0 ? 0.0 : sim_frame(c, (int)c->xquat.size() / 4 + s)[FR_QUAT + k];
}
void cassie_sim_body_contact_force(const cassie_sim_t *c, double cfrc[6], const char *name) {
  const int b = sim_body(c, name, "cassie_sim_body_contact_force");
  for (int k = 0; k < 6; k++) cfrc[k] = b < 0 ? 0.0 : sim_frame(c, b)[FR_CFRC + k];
}
static void sim_jacobian(cassie_sim_t *c, int f, double *jac, double *jac_rot) {
  const int nv = c->b->impl->hm.nv;
  if (f < 0) { for (int i = 0; i < 3 * nv; i++) { jac[i] = 0; if (jac_rot) jac_rot[i] = 0; } return; }
  sim_push(c); c->b->impl->frame_jacobian(f, jac, jac_rot);
}
void cassie_sim_get_jacobian(cassie_sim_t *c, double *jac, const char *name) { sim_jacobian(c, sim_body(c, name, "cassie_sim_get_jacobian"), jac, nullptr); }
void cassie_sim_get_jacobian_full(cassie_sim_t *c, double *jac, double *jac_rot, const char *name) { sim_jacobian(c, sim_body(c, name, "cassie_sim_get_jacobian_full"), jac, jac_rot); }
void cassie_sim_get_jacobian_full_site(cassie_sim_t *c, double *jac, double *jac_rot, const char *name) {
  const int s = sim_site(c, name, "cassie_sim_get_jacobian_full_site");
  sim_jacobian(c, s < 0 ? -1 : (int)c->xquat.size() / 4 + s, jac, jac_rot);
}
// ---- dynamics (src/cassiemujoco.c:1647-1749): one dynamics launch at the CURRENT state, then host arithmetic.  The reference's mj_fwdPosition there also
// rewrites d->xpos & co.; the mirrors keep the last step's poses, as with the Jacobians.  M is [nv][nv] (nv = 32, or 38 with the extra free body).
static bool sim_dynamics(const cassie_sim_t *cc, std::vector<double> &M, std::vector<double> *J, std::vector<double> *err, double *Icm) {
  cassie_sim_t *c = const_cast<cassie_sim_t *>(cc); sim_push(c);
  const int nv = c->b->impl->hm.nv, ne = 3 * c->b->impl->hm.neq;
  M.assign((size_t)nv * nv, 0.0); if (J) J->assign((size_t)ne * nv, 0.0); if (err) err->assign(ne, 0.0);
  return c->b->impl->dynamics() && c->b->impl->get_dynamics(M.data(), nullptr, J ? J->data() : nullptr, err ? err->data() : nullptr, Icm);
}
void cassie_sim_full_mass_matrix(const cassie_sim_t *c, double M[1024]) {
  std::vector<double> F; const int nv = c->b->impl->hm.nv; sim_dynamics(c, F, nullptr, nullptr, nullptr);
  for (int i = 0; i < 32; i++) for (int j = 0; j < 32; j++) M[i * 32 + j] = F[(size_t)i * nv + j];
}
void cassie_sim_minimal_mass_matrix(const cassie_sim_t *c, double M[256]) {
  static const int IND[16] = {0, 1, 2, 3, 4, 5, 6, 7, 8, 12, 18, 19, 20, 21, 25, 31};   // the floating base, then the 10 motors
  std::vector<double> F; const int nv = c->b->impl->hm.nv; sim_dynamics(c, F, nullptr, nullptr, nullptr);
  for (int i = 0; i < 16; i++) for (int j = 0; j < 16; j++) M[i * 16 + j] = F[(size_t)IND[i] * nv + IND[j]];
}
// the reference picks the rows of the equalities named left- / right-achilles-rod-eq; the compiled model keeps no equality names, so the connects are
// picked by their body1 instead (the same rows in the models that name them)
void cassie_sim_loop_constraint_info(const cassie_sim_t *c, double J_cl[192], double err_cl[6]) {
  for (int i = 0; i < 192; i++) J_cl[i] = 0; for (int i = 0; i < 6; i++) err_cl[i] = 0;
  const HostModel &hm = c->b->impl->hm; const int nv = hm.nv, lb = hm.body_id("left-achilles-rod"), rb = hm.body_id("right-achilles-rod");
  std::vector<int> eqs; for (int e = 0; e < hm.neq; e++) if (hm.eq_obj1id[e] >= 0 && (hm.eq_obj1id[e] == lb || hm.eq_obj1id[e] == rb)) eqs.push_back(e);
  if (eqs.empty()) { set_err("cassie_sim_loop_constraint_info: no connect equality on left- / right-achilles-rod"); return; }
  std::vector<double> F, J, err; if (!sim_dynamics(c, F, &J, &err, nullptr)) return;
  int row = 0;
  for (int e : eqs) for (int k = 0; k < 3 && row < 6; k++, row++) {
    for (int j = 0; j < 32; j++) J_cl[row * 32 + j] = J[(size_t)(3 * e + k) * nv + j];
    err_cl[row] = err[3 * e + k];
  }
}
void cassie_sim_centroid_inertia(const cassie_sim_t *c, double Icm[9]) {
  std::vector<double> F; for (int i = 0; i < 9; i++) Icm[i] = 0;
  sim_dynamics(c, F, nullptr, nullptr, Icm);
}
// pose 2 in the frame of pose 1: mju_negPose, then mju_mulPose (host arithmetic, unit quaternions)
void cassie_sim_relative_pose(double pos1[3], double quat1[4], double pos2[3], double quat2[4], double pos2_in_pos1[3], double quat2_in_quat1[4]) {
  const double w = quat1[0], x = -quat1[1], y = -quat1[2], z = -quat1[3];   // the conjugate of quat1 and its rotation matrix
  const double R[9] = {1 - 2 * (y * y + z * z), 2 * (x * y - w * z), 2 * (x * z + w * y), 2 * (x * y + w * z), 1 - 2 * (x * x + z * z), 2 * (y * z - w * x),
                       2 * (x * z - w * y), 2 * (y * z + w * x), 1 - 2 * (x * x + y * y)};
  const double *q = quat2, d[3] = {pos2[0] - pos1[0], pos2[1] - pos1[1], pos2[2] - pos1[2]};
  double r[4] = {w * q[0] - x * q[1] - y * q[2] - z * q[3], w * q[1] + x * q[0] + y * q[3] - z * q[2], w * q[2] - x * q[3] + y * q[0] + z * q[1], w * q[3] + x * q[2] - y * q[1] + z * q[0]};
  for (int k = 0; k < 4; k++) quat2_in_quat1[k] = r[k];
  for (int k = 0; k < 3; k++) pos2_in_pos1[k] = R[3 * k] * d[0] + R[3 * k + 1] * d[1] + R[3 * k + 2] * d[2];   // R (pos2 - pos1) = R pos2 + (-R pos1)
}
// ---- model constants (domain randomisation).  include/cassiemujoco.h / src/cassiemujoco.c:1303-1436: the reference hands out pointers into
// its private mjModel copy; here they point into host mirrors that are uploaded before the next step / query / set_const.
void cassie_sim_params(cassie_sim_t *c, int *params) { const HostModel &hm = c->b->impl->hm; params[0] = hm.nq; params[1] = hm.nv; params[2] = hm.nu; params[3] = 29; params[4] = hm.nbody; params[5] = hm.ngeom; }
double *cassie_sim_dof_damping(cassie_sim_t *c) { return c->m_damp.data(); }
double *cassie_sim_body_mass(cassie_sim_t *c) { return c->m_mass.data(); }
double *cassie_sim_body_ipos(cassie_sim_t *c) { return c->m_ipos.data(); }
double *cassie_sim_geom_friction(cassie_sim_t *c) { return c->m_fric.data(); }
void cassie_sim_set_dof_damping(cassie_sim_t *c, double *damp) { for (size_t i = 0; i < c->m_damp.size(); i++) c->m_damp[i] = damp[i]; }
void cassie_sim_set_body_mass(cassie_sim_t *c, double *mass) { for (size_t i = 0; i < c->m_mass.size(); i++) c->m_mass[i] = mass[i]; }
void cassie_sim_set_body_ipos(cassie_sim_t *c, double *ipos) {   // the reference indexes its argument with [i + j], not [3 i + j] (:1386-1393); kept
  const int nb = (int)c->m_mass.size(); for (int i = 0; i < nb; i++) for (int j = 0; j < 3; j++) c->m_ipos[3 * i + j] = ipos[i + j]; }
void cassie_sim_set_geom_friction(cassie_sim_t *c, double *fric) { for (size_t i = 0; i < c->m_fric.size(); i++) c->m_fric[i] = fric[i]; }
void cassie_sim_set_body_name_mass(cassie_sim_t *c, const char *name, double mass) { const int id = c->b->impl->hm.body_id(name ? name : ""); if (id >= 0) c->m_mass[id] = mass; }
double cassie_sim_get_body_name_mass(cassie_sim_t *c, const char *name) { const int id = c->b->impl->hm.body_id(name ? name : ""); return id >= 0 ? c->m_mass[id] : 0.0; }
void cassie_sim_set_body_name_ipos(cassie_sim_t *c, const char *name, double *ipos) { const int id = c->b->impl->hm.body_id(name ? name : ""); if (id >= 0) for (int k = 0; k < 3; k++) c->m_ipos[3 * id + k] = ipos[k]; }
double *cassie_sim_get_body_name_ipos(cassie_sim_t *c, const char *name) { const int id = c->b->impl->hm.body_id(name ? name : ""); return id >= 0 ? &c->m_ipos[3 * id] : nullptr; }
// src/cassiemujoco.c:1408-1418: a body's position in its parent frame through the host mirror (uploaded before the next launch); any body is accepted,
// the world body's and the extra free body's entries have no effect, as in MuJoCo.  An unknown name: NULL / no change, and an error (the reference indexes -1)
double *cassie_sim_get_body_name_pos(cassie_sim_t *c, const char *name) {
  const int id = c->b->impl->hm.body_id(name ? name : "");
  if (id < 0) { set_err(std::string("cassie_sim_get_body_name_pos: unknown body ") + (name ? name : "(null)")); return nullptr; }
  return &c->m_bpos[3 * id];
}
void cassie_sim_set_body_name_pos(cassie_sim_t *c, const char *name, double *data) {
  double *p = cassie_sim_get_body_name_pos(c, name);
  if (p && data) for (int k = 0; k < 3; k++) p[k] = data[k];
}
// src/cassiemujoco.c:2114-2192: the delay line and the encoders' filters, read and written through the simulator's batch (pending writes through
// the borrowed mirrors go first)
void cassie_sim_torque_delay(cassie_sim_t *c, double *t) { sim_push(c); c->b->impl->get_actuator_state(t, nullptr, nullptr, nullptr); }
void cassie_sim_set_torque_delay(cassie_sim_t *c, double *t) { sim_push(c); c->b->impl->set_actuator_state(t, nullptr, nullptr, nullptr, nullptr); }
void cassie_sim_get_joint_filter(cassie_sim_t *c, double *x, double *y) { sim_push(c); c->b->impl->get_actuator_state(nullptr, nullptr, x, y); }
void cassie_sim_set_joint_filter(cassie_sim_t *c, double *x, double *y) { sim_push(c); c->b->impl->set_actuator_state(nullptr, nullptr, x, y, nullptr); if (c->act_lent) sim_pull_act(c); }
void cassie_sim_get_drive_filter(cassie_sim_t *c, int *x) { sim_push(c); c->b->impl->get_actuator_state(nullptr, x, nullptr, nullptr); }
void cassie_sim_set_drive_filter(cassie_sim_t *c, int *x) { sim_push(c); c->b->impl->set_actuator_state(nullptr, x, nullptr, nullptr, nullptr); if (c->act_lent) sim_pull_act(c); }
void *cassie_sim_joint_filter(cassie_sim_t *c) { sim_lend_act(c); return &c->jfilt[0][0]; }   // joint_filter_t[6]
void *cassie_sim_drive_filter(cassie_sim_t *c) { sim_lend_act(c); return &c->dfilt[0][0]; }   // drive_filter_t[10]
// :1237: mjData's ctrl as the last physics step applied it; writes through the pointer have no effect (cassie_motor_data overwrites d->ctrl before
// mj_step in the reference); zeros after cassie_sim_full_reset until the next step
double *cassie_sim_ctrl(cassie_sim_t *c) { sim_lend_act(c); return c->ctrl; }
int cassie_sim_get_joint_num_dof(cassie_sim_t *c, const char *name) { const HostModel &hm = c->b->impl->hm; const int j = hm.joint_id(name ? name : ""); if (j < 0) return 0; return hm.jnt_type[j] == JNT_FREE ? 6 : (hm.jnt_type[j] == JNT_BALL ? 3 : 1); }
void cassie_sim_set_dof_name_damping(cassie_sim_t *c, const char *name, double *damp) { const HostModel &hm = c->b->impl->hm; const int j = hm.joint_id(name ? name : ""); if (j < 0) return; const int nd = cassie_sim_get_joint_num_dof(c, name); for (int i = 0; i < nd; i++) c->m_damp[hm.jnt_dofadr[j] + i] = damp[i]; }
double *cassie_sim_get_dof_name_damping(cassie_sim_t *c, const char *name) { const HostModel &hm = c->b->impl->hm; const int j = hm.joint_id(name ? name : ""); return j >= 0 ? &c->m_damp[hm.jnt_dofadr[j]] : nullptr; }
// the reference copies 3 values to &geom_friction[geom_id] (:1417-1421, not 3 * geom_id); here the geom's own triple is addressed
void cassie_sim_set_geom_name_friction(cassie_sim_t *c, const char *name, double *fric) { const int g = c->b->impl->hm.geom_id(name ? name : ""); if (g >= 0) for (int k = 0; k < 3; k++) c->m_fric[3 * g + k] = fric[k]; }
double *cassie_sim_get_geom_name_friction(cassie_sim_t *c, const char *name) { const int g = c->b->impl->hm.geom_id(name ? name : ""); return g >= 0 ? &c->m_fric[3 * g] : nullptr; }
void cassie_sim_just_set_const(cassie_sim_t *c) { sim_push(c); cassie_batch_set_const(c->b, nullptr, 0); }
void cassie_sim_set_const(cassie_sim_t *c) { sim_push(c); cassie_batch_set_const(c->b, nullptr, 1); sim_pull(c); }
void cassie_sim_full_reset(cassie_sim_t *c) {
  // src/cassiemujoco.c:2008-2033: qpos <- 35 constants, zero qvel / ctrl / applied forces / qacc, zero the torque delay line.
  // It does NOT touch time, the encoder filters or cassie_out, and does not call mj_forward.
  static const double q[35] = {0, 0, 1.01, 1, 0, 0, 0, 0.0045, 0, 0.4973, 0.9785, -0.0164, 0.01787, -0.2049, -1.1997, 0, 1.4267, 0, -1.5244, 1.5244, -1.5968,
                               -0.0045, 0, 0.4973, 0.9786, 0.00386, -0.01524, -0.2051, -1.1997, 0, 1.4267, 0, -1.5244, 1.5244, -1.5968};
  std::vector<double> cst(CST_W); c->b->impl->get("cst", cst.data());
  for (int i = 0; i < 60; i++) cst[CS_DELAY + i] = 0;
  c->b->impl->set("cst", cst.data());
  memcpy(c->qpos, q, sizeof q); memset(c->qvel, 0, sizeof c->qvel);   // 35 entries only (:2025): qpos beyond them (the cup of cassie_tray_box.xml) keeps its values
  c->b->impl->set("qpos", c->qpos); c->b->impl->set("qvel", c->qvel); cassie_batch_clear_forces(c->b);
  if (c->b->impl->dev_ptr("applied")) { const std::vector<double> zero(c->b->impl->hm.nv, 0.0); c->b->impl->set_applied_forces(nullptr, zero.data(), nullptr); }   // qfrc_applied <- 0 (:2024)
  if (!c->acc.empty()) {   // qacc <- 0 (:2025): what the reference's query then gives, with qvel = qacc = 0, is cacc = (0, 0, 0, -g) for every body
    const HostModel &hm = c->b->impl->hm; std::vector<double> row(c->acc.size(), 0.0);
    for (int b = 0; b < (int)c->xquat.size() / 4; b++) for (int k = 0; k < 3; k++) row[AC_CACC + AC_SLOT * b + 3 + k] = -hm.gravity[k];
    c->b->impl->set("acc", row.data());
  }
  c->b->impl->reset_estimator(nullptr); c->b->impl->reset_estimator_device(nullptr);   // state_output_setup (src/cassiemujoco.c:2032) restarts the estimator's filters
  c->ctrl_zero = true;   // ctrl <- 0 (:2024) until the next step applies one
  sim_pull(c);
}
// sizes the reference's Python wrapper asks for (src/cassiemujoco.c:1038-1060)
int cassie_sim_nbody(const cassie_sim_t *c) { return c->b->impl->hm.nbody; }
int cassie_sim_ngeom(const cassie_sim_t *c) { return c->b->impl->hm.ngeom; }
int cassie_sim_njnt(const cassie_sim_t *c) { return c->b->impl->hm.njnt; }
int cassie_sim_nu(const cassie_sim_t *c) { return c->b->impl->hm.nu; }
// src/cassiemujoco.c:1183-1189: qpos += h * qvel on the joint manifold; the reference then feeds an uninitialised cassie_out_t to its estimator,
// so *y carries no information there -- it is zeroed here
void cassie_integrate_pos(cassie_sim_t *c, state_out_t *y) { sim_push(c); cassie_batch_integrate_pos(c->b); c->b->impl->sync(); sim_pull(c); if (y) memset(y, 0, sizeof *y); }

// ---- geom placement (src/cassiemujoco.c:1466-1541; example/test_terrain.c:118-157 moves the stair boxes with these): borrowed pointers into host
// mirrors in the reference's geom numbering; the constant block is rebuilt before the next launch.  As in MuJoCo a new size leaves geom_rbound alone.
double *cassie_sim_geom_pos(cassie_sim_t *c) { return c->m_gpos.data(); }
double *cassie_sim_geom_quat(cassie_sim_t *c) { return c->m_gquat.data(); }
double *cassie_sim_geom_size(cassie_sim_t *c) { return c->m_gsize.data(); }
double *cassie_sim_geom_name_pos(cassie_sim_t *c, const char *name) { const int g = c->b->impl->hm.geom_id(name ? name : ""); return g >= 0 ? &c->m_gpos[3 * g] : nullptr; }
double *cassie_sim_geom_name_quat(cassie_sim_t *c, const char *name) { const int g = c->b->impl->hm.geom_id(name ? name : ""); return g >= 0 ? &c->m_gquat[4 * g] : nullptr; }
double *cassie_sim_geom_name_size(cassie_sim_t *c, const char *name) { const int g = c->b->impl->hm.geom_id(name ? name : ""); return g >= 0 ? &c->m_gsize[3 * g] : nullptr; }
void cassie_sim_set_geom_pos(cassie_sim_t *c, double *pos) { for (size_t i = 0; i < c->m_gpos.size(); i++) c->m_gpos[i] = pos[i]; }
void cassie_sim_set_geom_quat(cassie_sim_t *c, double *quat) { for (size_t i = 0; i < c->m_gquat.size(); i++) c->m_gquat[i] = quat[i]; }
void cassie_sim_set_geom_size(cassie_sim_t *c, double *size) { for (size_t i = 0; i < c->m_gsize.size(); i++) c->m_gsize[i] = size[i]; }
void cassie_sim_set_geom_name_pos(cassie_sim_t *c, const char *name, double *pos) { double *p = cassie_sim_geom_name_pos(c, name); if (p) for (int k = 0; k < 3; k++) p[k] = pos[k]; }
void cassie_sim_set_geom_name_quat(cassie_sim_t *c, const char *name, double *quat) { double *p = cassie_sim_geom_name_quat(c, name); if (p) for (int k = 0; k < 4; k++) p[k] = quat[k]; }
void cassie_sim_set_geom_name_size(cassie_sim_t *c, const char *name, double *size) { double *p = cassie_sim_geom_name_size(c, name); if (p) for (int k = 0; k < 3; k++) p[k] = size[k]; }
// the same for a batch: one placement shared by all its environments (pos / quat / size: NULL leaves that part alone); 0 / -1 (unknown geom)
int cassie_batch_set_geom_pose(cassie_batch_t *b, const char *name, const double *pos, const double *quat, const double *size) {
  HostModel &hm = b->impl->hm; const int g = hm.geom_id(name ? name : "");
  if (g < 0) { set_err("cassie_batch_set_geom_pose: unknown geom"); return -1; }
  if (pos) for (int k = 0; k < 3; k++) hm.geom_pos[3 * g + k] = pos[k];
  if (quat) for (int k = 0; k < 4; k++) hm.geom_quat[4 * g + k] = quat[k];
  if (size) for (int k = 0; k < 3; k++) hm.geom_size[3 * g + k] = size[k];
  return b->impl->rebuild_model() && b->impl->shared_geom_changed(g) ? 0 : -1;   // per-environment rows, if any, take the shared placement of this geom
}
// per-environment placement of a static plane / box (extends src/cassiemujoco.c:1466-1541 to one placement per environment); see include/cassie_b200.h
int cassie_batch_set_env_geom_pose(cassie_batch_t *b, const char *name, const double *pos, const double *quat, const double *size, const unsigned char *mask) {
  return b->impl->set_env_geom(b->impl->hm.geom_id(name ? name : ""), pos, quat, size, mask) ? 0 : -1;
}
int cassie_batch_get_env_geom_pose(cassie_batch_t *b, const char *name, double *pos, double *quat, double *size) {
  return b->impl->get_env_geom(b->impl->hm.geom_id(name ? name : ""), pos, quat, size) ? 0 : -1;
}
int cassie_batch_clear_env_geom_poses(cassie_batch_t *b) { return b->impl->clear_env_geoms() ? 0 : -1; }
// per-environment terrain (bank entry, height-field position and size); see include/cassie_b200.h
int cassie_batch_set_env_hfield(cassie_batch_t *b, const int *terrain, const double *pos, const double *size, const unsigned char *mask) { return b->impl->set_env_hfield(terrain, pos, size, mask) ? 0 : -1; }
int cassie_batch_get_env_hfield(cassie_batch_t *b, int *terrain, double *pos, double *size) { return b->impl->get_env_hfield(terrain, pos, size) ? 0 : -1; }
int cassie_batch_clear_env_hfield(cassie_batch_t *b) { return b->impl->clear_env_hfield() ? 0 : -1; }
// per-environment body offsets; see include/cassie_b200.h
int cassie_batch_set_env_body_pos(cassie_batch_t *b, const double *pos, const unsigned char *mask) { return b->impl->set_env_body_pos(pos, mask) ? 0 : -1; }
int cassie_batch_get_env_body_pos(cassie_batch_t *b, double *pos) { return b->impl->get_env_body_pos(pos) ? 0 : -1; }
int cassie_batch_clear_env_body_pos(cassie_batch_t *b) { return b->impl->clear_env_body_pos() ? 0 : -1; }
// per-environment actuators and the controller-stage state; see include/cassie_b200.h
int cassie_batch_set_env_actuators(cassie_batch_t *b, const double *ctrlrange, const double *rpm, const int *delay, const unsigned char *mask) { return b->impl->set_env_actuators(ctrlrange, rpm, delay, mask) ? 0 : -1; }
int cassie_batch_get_env_actuators(cassie_batch_t *b, double *ctrlrange, double *rpm, int *delay) { return b->impl->get_env_actuators(ctrlrange, rpm, delay) ? 0 : -1; }
int cassie_batch_clear_env_actuators(cassie_batch_t *b) { return b->impl->clear_env_actuators() ? 0 : -1; }
// per-environment mechanics (link inertia, rotor armature, hinge springs); see include/cassie_b200.h
int cassie_batch_set_env_mechanics(cassie_batch_t *b, const double *inertia, const double *armature, const double *stiffness, const double *springref, const unsigned char *mask) {
  return b->impl->set_env_mechanics(inertia, armature, stiffness, springref, mask) ? 0 : -1; }
int cassie_batch_get_env_mechanics(cassie_batch_t *b, double *inertia, double *armature, double *stiffness, double *springref) { return b->impl->get_env_mechanics(inertia, armature, stiffness, springref) ? 0 : -1; }
int cassie_batch_clear_env_mechanics(cassie_batch_t *b) { return b->impl->clear_env_mechanics() ? 0 : -1; }
// per-environment contact softness (solref, solimp, solmix per collision geom); see include/cassie_b200.h
int cassie_batch_set_env_contact(cassie_batch_t *b, const double *solref, const double *solimp, const double *solmix, const unsigned char *mask) {
  return b->impl->set_env_contact(solref, solimp, solmix, mask) ? 0 : -1; }
int cassie_batch_get_env_contact(cassie_batch_t *b, double *solref, double *solimp, double *solmix) { return b->impl->get_env_contact(solref, solimp, solmix) ? 0 : -1; }
int cassie_batch_clear_env_contact(cassie_batch_t *b) { return b->impl->clear_env_contact() ? 0 : -1; }
// per-environment applied forces (xfrc_applied per body, qfrc_applied per dof); see include/cassie_b200.h
int cassie_batch_set_applied_forces(cassie_batch_t *b, const double *xfrc, const double *qfrc, const unsigned char *mask) { return b->impl->set_applied_forces(xfrc, qfrc, mask) ? 0 : -1; }
int cassie_batch_get_applied_forces(cassie_batch_t *b, double *xfrc, double *qfrc) { return b->impl->get_applied_forces(xfrc, qfrc) ? 0 : -1; }
int cassie_batch_enable_applied_forces(cassie_batch_t *b, int on) { return b->impl->enable_applied_forces(on != 0) ? 0 : -1; }
// per-tick traces of step launches; see include/cassie_b200.h
int cassie_batch_set_trace(cassie_batch_t *b, const int *source, const int *column, int k, int max_ticks) { return b->impl->set_trace(source, column, k, max_ticks) ? 0 : -1; }
int cassie_batch_trace_ticks(const cassie_batch_t *b) { return b->impl->trace_ticks(); }
int cassie_batch_get_trace(cassie_batch_t *b, double *out) { return b->impl->get_trace(out) ? 0 : -1; }
// contact lists of step and forward launches; see include/cassie_b200.h
int cassie_batch_enable_contacts(cassie_batch_t *b, int on) { return b->impl->enable_contacts(on != 0) ? 0 : -1; }
int cassie_batch_get_contacts(cassie_batch_t *b, double *out) { return b->impl->get_contacts(out) ? 0 : -1; }
// sensor models drawn in the step kernel; see include/cassie_b200.h
int cassie_batch_set_env_sensors(cassie_batch_t *b, const double *enc_offset, const double *enc_noise, const double *imu_quat, const double *imu_bias, const double *imu_noise, const unsigned char *mask) {
  return b->impl->set_env_sensors(enc_offset, enc_noise, imu_quat, imu_bias, imu_noise, mask) ? 0 : -1; }
int cassie_batch_get_env_sensors(cassie_batch_t *b, double *enc_offset, double *enc_noise, double *imu_quat, double *imu_bias, double *imu_noise) { return b->impl->get_env_sensors(enc_offset, enc_noise, imu_quat, imu_bias, imu_noise) ? 0 : -1; }
int cassie_batch_clear_env_sensors(cassie_batch_t *b) { return b->impl->clear_env_sensors() ? 0 : -1; }
int cassie_batch_seed_sensors(cassie_batch_t *b, unsigned long long seed, const unsigned char *mask) { return b->impl->seed_sensors(seed, mask) ? 0 : -1; }
int cassie_batch_get_sensor_rng(cassie_batch_t *b, unsigned long long *seed, unsigned long long *counter) { return b->impl->get_sensor_rng(seed, counter) ? 0 : -1; }
// names of the compiled model's objects (mj_name2id / mj_id2name for the kinds it keeps names of); see include/cassie_b200.h
int cassie_batch_name2id(const cassie_batch_t *b, const char *type, const char *name) {
  const std::vector<std::string> *t = name_table(b->impl->hm, type, "cassie_batch_name2id");
  if (!t || !name || !*name) return -1;
  for (int i = 0; i < (int)t->size(); i++) if ((*t)[i] == name) return i;
  return -1;
}
const char *cassie_batch_id2name(const cassie_batch_t *b, const char *type, int id) {
  const std::vector<std::string> *t = name_table(b->impl->hm, type, "cassie_batch_id2name");
  if (!t || id < 0 || id >= (int)t->size() || (*t)[id].empty()) return nullptr;
  return (*t)[id].c_str();
}
int cassie_sim_mj_name2id(cassie_sim_t *c, char *mj_type, char *name) { return cassie_batch_name2id(c->b, mj_type, name); }
int cassie_batch_get_actuator_state(cassie_batch_t *b, double *torque_delay, int *drive_filter, double *joint_x, double *joint_y) { return b->impl->get_actuator_state(torque_delay, drive_filter, joint_x, joint_y) ? 0 : -1; }
int cassie_batch_set_actuator_state(cassie_batch_t *b, const double *torque_delay, const int *drive_filter, const double *joint_x, const double *joint_y, const unsigned char *mask) {
  return b->impl->set_actuator_state(torque_delay, drive_filter, joint_x, joint_y, mask) ? 0 : -1; }
int cassie_batch_set_hfield_size(cassie_batch_t *b, const double size[4]) { return b->impl->set_hfield_size(size) ? 0 : -1; }
int cassie_batch_get_hfield_size(const cassie_batch_t *b, double size[4]) {
  const HostModel &hm = b->impl->hm;
  if (hm.nhfield != 1) { set_err("cassie_batch_get_hfield_size: this model has no height field"); return -1; }
  if (size) for (int c = 0; c < 4; c++) size[c] = hm.hfield_size[c];
  return 0;
}
int cassie_batch_set_frames(cassie_batch_t *b, const char *const *names, const int *kinds, int count) { return b->impl->set_frames(names, kinds, count) ? 0 : -1; }
int cassie_batch_nframes(const cassie_batch_t *b) { return (int)(b->impl->frame_list.size() / 2); }
int cassie_batch_get_frames(cassie_batch_t *b, double *out) { return b->impl->get("frames", out) ? 0 : -1; }
int cassie_batch_frame_jacobian(cassie_batch_t *b, int frame, double *jacp, double *jacr) { return b->impl->frame_jacobian(frame, jacp, jacr) ? 0 : -1; }
int cassie_batch_set_rays(cassie_batch_t *b, const int *frame, const double *origin, const double *dir, const double *max_dist, int k) { return b->impl->set_rays(frame, origin, dir, max_dist, k) ? 0 : -1; }
int cassie_batch_nrays(const cassie_batch_t *b) { return b->impl->nray; }
int cassie_batch_raycast(cassie_batch_t *b) { return b->impl->raycast() ? 0 : -1; }
int cassie_batch_get_rays(cassie_batch_t *b, double *out) { return b->impl->get_rays(out) ? 0 : -1; }
// the index of a fixed <camera> of the model, or -1 with the error recorded under `verb`
static int fixed_camera(const HostModel &hm, const char *camera, const char *verb) {
  const int k = camera ? hm.camera_id(camera) : -1;
  if (k < 0) {
    std::string names; for (const std::string &c : hm.names_camera) names += (names.empty() ? "" : ", ") + c;
    set_err(std::string(verb) + ": unknown camera '" + std::string(camera ? camera : "") + "' (the model's cameras: " + (names.empty() ? "none" : names) + ")"); return -1;
  }
  if (hm.camera_mode[k] != CAM_FIXED) { set_err(std::string(verb) + ": camera '" + std::string(camera) + "' is not a fixed camera (track / target modes are not rendered)"); return -1; }
  return k;
}
int cassie_batch_set_camera(cassie_batch_t *b, const char *camera, int width, int height, double zfar) {
  const HostModel &hm = b->impl->hm;
  if (width == 0) return b->impl->set_cameras(0, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, "cassie_batch_set_camera", false) ? 0 : -1;
  const int k = fixed_camera(hm, camera, "cassie_batch_set_camera");
  if (k < 0) return -1;
  return b->impl->set_cameras(1, &hm.camera_body[k], &hm.camera_pos[3 * k], &hm.camera_quat[4 * k], &hm.camera_fovy[k], width, height, zfar, "cassie_batch_set_camera", false) ? 0 : -1;
}
int cassie_batch_set_camera_mount(cassie_batch_t *b, const char *body, const double pos[3], const double quat[4], double fovy, int width, int height, double zfar) {
  if (width == 0) return b->impl->set_cameras(0, nullptr, nullptr, nullptr, nullptr, 0, 0, 0, "cassie_batch_set_camera_mount", false) ? 0 : -1;
  const int id = body ? b->impl->hm.body_id(body) : -1;
  if (id < 0) { set_err("cassie_batch_set_camera_mount: unknown body '" + std::string(body ? body : "") + "'"); return -1; }
  return b->impl->set_cameras(1, &id, pos, quat, &fovy, width, height, zfar, "cassie_batch_set_camera_mount", false) ? 0 : -1;
}
int cassie_batch_set_cameras(cassie_batch_t *b, int k, const int *body, const double *pos, const double *quat, const double *fovy, int width, int height, double zfar) {
  return b->impl->set_cameras(k, body, pos, quat, fovy, width, height, zfar, "cassie_batch_set_cameras", true) ? 0 : -1;
}
int cassie_batch_model_camera(cassie_batch_t *b, const char *camera, int *body, double pos[3], double quat[4], double *fovy) {
  const HostModel &hm = b->impl->hm;
  const int k = fixed_camera(hm, camera, "cassie_batch_model_camera");
  if (k < 0) return -1;
  if (body) *body = hm.camera_body[k];
  if (pos) for (int i = 0; i < 3; i++) pos[i] = hm.camera_pos[3 * k + i];
  if (quat) for (int i = 0; i < 4; i++) quat[i] = hm.camera_quat[4 * k + i];
  if (fovy) *fovy = hm.camera_fovy[k];
  return 0;
}
int cassie_batch_ncameras(const cassie_batch_t *b) { return b->impl->cam.k; }
int cassie_batch_set_env_cameras(cassie_batch_t *b, const double *pos, const double *quat, const double *fovy, const unsigned char *mask) { return b->impl->set_env_cameras(pos, quat, fovy, mask) ? 0 : -1; }
int cassie_batch_get_env_cameras(cassie_batch_t *b, double *pos, double *quat, double *fovy) { return b->impl->get_env_cameras(pos, quat, fovy) ? 0 : -1; }
int cassie_batch_clear_env_cameras(cassie_batch_t *b) { return b->impl->clear_env_cameras() ? 0 : -1; }
int cassie_batch_enable_camera_geoms(cassie_batch_t *b, int on) { return b->impl->enable_camera_geoms(on != 0) ? 0 : -1; }
int cassie_batch_get_camera_geoms(cassie_batch_t *b, int *out) { return b->impl->get_camera_geoms(out) ? 0 : -1; }
int cassie_batch_render_depth(cassie_batch_t *b) { return b->impl->render_depth() ? 0 : -1; }
int cassie_batch_get_depth(cassie_batch_t *b, double *out) { return b->impl->get_depth(out) ? 0 : -1; }
int cassie_batch_dynamics(cassie_batch_t *b) { return b->impl->dynamics() ? 0 : -1; }
int cassie_batch_get_dynamics(cassie_batch_t *b, double *M, double *bias, double *J_eq, double *eq_err, double *Icm) { return b->impl->get_dynamics(M, bias, J_eq, eq_err, Icm) ? 0 : -1; }
int cassie_batch_inverse(cassie_batch_t *b, const double *qacc) { return b->impl->inverse(qacc) ? 0 : -1; }
int cassie_batch_get_inverse(cassie_batch_t *b, double *qfrc_inverse, double *qfrc_constraint, int *counts) { return b->impl->get_inverse(qfrc_inverse, qfrc_constraint, counts) ? 0 : -1; }
int cassie_batch_neq(const cassie_batch_t *b) { return b->impl->hm.neq; }
int cassie_batch_enable_accelerations(cassie_batch_t *b, int on) { return b->impl->enable_accelerations(on != 0) ? 0 : -1; }
int cassie_batch_get_accelerations(cassie_batch_t *b, double *qacc, double *cacc) { return b->impl->get_accelerations(qacc, cacc) ? 0 : -1; }

// ---- legacy verbs RL wrappers call around cassie_sim_step_pd (src/cassiemujoco.c:1072-1093, 1137-1145, 1159-1181, 1196-1225, 1974-2000, 2086-2092, 3380-3452)
// the dynamic subset of cassie_out_t from an observation row, the rest as cassie_out_init leaves it (:672-734)
static void fill_cassie_out(const double *o, const double *radio, cassie_out_t *y) {
  memset(y, 0, sizeof *y);
  y->isCalibrated = true;
  y->pelvis.medullaCounter = 1; y->pelvis.medullaCpuLoad = 159; y->pelvis.vtmTemperature = 40;
  y->pelvis.targetPc.etherCatStatus[1] = 8; y->pelvis.targetPc.etherCatStatus[4] = 1; y->pelvis.targetPc.taskExecutionTime = 2e-4; y->pelvis.targetPc.cpuTemperature = 60;
  y->pelvis.battery.dataGood = true; y->pelvis.battery.stateOfCharge = 1;
  for (int i = 0; i < 4; i++) y->pelvis.battery.temperature[i] = 30;
  for (int i = 0; i < 12; i++) y->pelvis.battery.voltage[i] = 4.2;
  y->pelvis.radio.radioReceiverSignalGood = true; y->pelvis.radio.receiverMedullaSignalGood = true;
  for (int i = 0; i < 16; i++) y->pelvis.radio.channel[i] = radio[i];
  y->pelvis.vectorNav.dataGood = true; y->pelvis.vectorNav.pressure = 101.325; y->pelvis.vectorNav.temperature = 25;
  for (int i = 0; i < 4; i++) y->pelvis.vectorNav.orientation[i] = o[OB_QUAT + i];
  for (int i = 0; i < 3; i++) { y->pelvis.vectorNav.angularVelocity[i] = o[OB_GYRO + i]; y->pelvis.vectorNav.linearAcceleration[i] = o[OB_ACCEL + i]; y->pelvis.vectorNav.magneticField[i] = o[OB_MAG + i]; }
  static const double tl[5] = {140.63, 140.63, 216.16, 216.16, 45.14}, gr[5] = {25, 25, 16, 16, 50};
  for (int sd = 0; sd < 2; sd++) {
    cassie_leg_out_t *leg = sd ? &y->rightLeg : &y->leftLeg; leg->medullaCounter = 1; leg->medullaCpuLoad = 94;
    elmo_out_t *dr[5] = {&leg->hipRollDrive, &leg->hipYawDrive, &leg->hipPitchDrive, &leg->kneeDrive, &leg->footDrive};
    for (int i = 0; i < 5; i++) { dr[i]->statusWord = 0x0637; dr[i]->dcLinkVoltage = 48; dr[i]->driveTemperature = 30; dr[i]->torqueLimit = tl[i]; dr[i]->gearRatio = gr[i];
      dr[i]->position = o[OB_MPOS + 5 * sd + i]; dr[i]->velocity = o[OB_MVEL + 5 * sd + i]; dr[i]->torque = o[OB_MTORQUE + 5 * sd + i]; }
    cassie_joint_out_t *jn[3] = {&leg->shinJoint, &leg->tarsusJoint, &leg->footJoint};
    for (int i = 0; i < 3; i++) { jn[i]->position = o[OB_JPOS + 3 * sd + i]; jn[i]->velocity = o[OB_JVEL + 3 * sd + i]; }
  }
}
// :2090-2092.  The observation row holds what `*y = c->cassie_out` copied out in the last step (:1127); before the first step it is the initial bus state
cassie_out_t cassie_sim_get_cassie_out(cassie_sim_t *c) { double o[OBS_W]; cassie_out_t y; c->b->impl->get("obs", o); fill_cassie_out(o, c->b->radio.data(), &y); return y; }
// :1137-1145: user torques -> safety layer -> motor model -> physics; y = the bus as the sensors filled it in this tick.  A pd_in_t that carries only
// motorPd.torque makes pd_input_step the identity on the torques, so the launch is the same one cassie_sim_step_pd uses
void cassie_sim_step(cassie_sim_t *c, cassie_out_t *y, const cassie_user_in_t *u) {
  pd_in_t pd; memset(&pd, 0, sizeof pd);
  for (int i = 0; i < 5; i++) { pd.leftLeg.motorPd.torque[i] = u->torque[i]; pd.rightLeg.motorPd.torque[i] = u->torque[5 + i]; }
  state_out_t so; sim_push(c); cassie_sim_step_pd_batch(c->b, &pd, &so); c->ctrl_zero = false; sim_pull(c);
  if (y) *y = cassie_sim_get_cassie_out(c);
}
// :1159-1181: the same tick with ONE physics step whatever the model's timestep is
void cassie_sim_step_pd_no2khz(cassie_sim_t *c, state_out_t *y, const pd_in_t *u) { sim_push(c); c->b->impl->nsub_override = 1; cassie_sim_step_pd_batch(c->b, u, y); c->b->impl->nsub_override = 0; c->ctrl_zero = false; sim_pull(c); }
// :1196-1204: the borrowed pointer is a host mirror, uploaded (constant block rebuilt) before the next launch
double *cassie_sim_timestep(cassie_sim_t *c) { return &c->timestep; }
void cassie_sim_set_timestep(cassie_sim_t *c, double dt) { c->timestep = dt; }
int cassie_batch_set_timestep(cassie_batch_t *b, double dt) { if (!(dt > 0)) return -1; b->impl->hm.timestep = dt; return b->impl->rebuild_model() ? 0 : -1; }
// :1221-1225
int cassie_sim_forward(cassie_sim_t *c) { sim_push(c); c->b->impl->step(0, 1); sim_pull(c); return 0; }
// :1974-2000: pin / free the pelvis with a stiff spring-damper on its three slides and damping on its ball joint
static void sim_hold(cassie_sim_t *c, bool on) {
  HostModel &hm = c->b->impl->hm; sim_push(c);
  for (int i = 0; i < 3 && i < hm.njnt; i++) { hm.jnt_stiffness[i] = on ? 1e5 : 0; if (on) hm.qpos_spring[i] = c->qpos[i]; }
  for (int i = 0; i < 6 && i < hm.nv; i++) { hm.dof_damping[i] = on ? (i < 3 ? 1e4 : 1e4) : 0; c->m_damp[i] = hm.dof_damping[i]; }
  c->b->impl->rebuild_model(); sim_push(c);
}
void cassie_sim_hold(cassie_sim_t *c) { sim_hold(c, true); }
void cassie_sim_release(cassie_sim_t *c) { sim_hold(c, false); }
// :3380-3452
cassie_state_t *cassie_state_alloc(void) { cassie_state *s = new cassie_state(); memset(s->qpos, 0, sizeof s->qpos); memset(s->qvel, 0, sizeof s->qvel); memset(s->qpos_snap, 0, sizeof s->qpos_snap); memset(s->qvel_snap, 0, sizeof s->qvel_snap); return s; }
void cassie_state_free(cassie_state_t *s) { if (!s) return; snap_delete(s->snap); delete s; }
double *cassie_state_time(cassie_state_t *s) { return &s->time; }
double *cassie_state_qpos(cassie_state_t *s) { return s->qpos; }
double *cassie_state_qvel(cassie_state_t *s) { return s->qvel; }
void cassie_get_state(const cassie_sim_t *cc, cassie_state_t *s) {
  cassie_sim_t *c = const_cast<cassie_sim_t *>(cc); BatchBase *impl = c->b->impl; sim_push(c);
  if (s->snap && !(s->snap->n == 1 && s->snap->qw == cassie_batch_row_width(c->b, "qpos") && s->snap->vw == cassie_batch_row_width(c->b, "qvel") && s->snap->device == impl->device)) { snap_delete(s->snap); s->snap = nullptr; }
  if (!s->snap) { s->snap = impl->snap_alloc(); if (!s->snap) return; }
  impl->snap_get(s->snap);
  memcpy(s->qpos, c->qpos, sizeof s->qpos); memcpy(s->qvel, c->qvel, sizeof s->qvel); s->time = c->time;
  memcpy(s->qpos_snap, s->qpos, sizeof s->qpos); memcpy(s->qvel_snap, s->qvel, sizeof s->qvel); s->time_snap = s->time; s->ctrl_zero = c->ctrl_zero;
}
void cassie_set_state(cassie_sim_t *c, const cassie_state_t *s) {
  if (!s->snap) { set_err("cassie_set_state: the state object holds no snapshot (cassie_get_state first)"); return; }
  if (!c->b->impl->snap_set(s->snap, nullptr)) return;   // any simulator of the same model accepts it
  c->ctrl_zero = s->ctrl_zero;   // mjData's ctrl is part of the reference's state
  memcpy(c->jfilt_dev, c->jfilt, sizeof c->jfilt); memcpy(c->dfilt_dev, c->dfilt, sizeof c->dfilt);   // the restored filters replace writes not yet uploaded
  sim_pull(c);
  // what the caller wrote through cassie_state_qpos / qvel / time after the snapshot was taken
  if (memcmp(s->qpos, s->qpos_snap, sizeof s->qpos)) memcpy(c->qpos, s->qpos, sizeof s->qpos);
  if (memcmp(s->qvel, s->qvel_snap, sizeof s->qvel)) memcpy(c->qvel, s->qvel, sizeof s->qvel);
  if (s->time != s->time_snap) c->time = s->time;
  sim_push(c);
}
void cassie_state_copy(cassie_state_t *dst, const cassie_state_t *src) {
  if (!src->snap) return;
  if (dst->snap && (dst->snap->n != src->snap->n || dst->snap->qw != src->snap->qw || dst->snap->vw != src->snap->vw || dst->snap->esz != src->snap->esz)) { snap_delete(dst->snap); dst->snap = nullptr; }
  if (!dst->snap) { dst->snap = snap_new(src->snap->device, src->snap->n, src->snap->esz, src->snap->qw, src->snap->vw); if (!dst->snap) return; }
  if (!snap_clone_into(dst->snap, src->snap)) { set_err("cassie_state_copy failed"); return; }
  memcpy(dst->qpos, src->qpos, sizeof dst->qpos); memcpy(dst->qvel, src->qvel, sizeof dst->qvel); dst->time = src->time;
  memcpy(dst->qpos_snap, src->qpos_snap, sizeof dst->qpos_snap); memcpy(dst->qvel_snap, src->qvel_snap, sizeof dst->qvel_snap); dst->time_snap = src->time_snap;
  dst->ctrl_zero = src->ctrl_zero;
}
cassie_state_t *cassie_state_duplicate(const cassie_state_t *src) { cassie_state_t *s = cassie_state_alloc(); cassie_state_copy(s, src); return s; }
// :1072-1093: model (per-environment constants, height field, timestep) and full dynamic state
void cassie_sim_copy(cassie_sim_t *dst, const cassie_sim_t *csrc) {
  cassie_sim_t *src = const_cast<cassie_sim_t *>(csrc); sim_push(src); sim_push(dst);
  if (!dst->b->impl->copy_model_from(src->b->impl)) return;
  dst->m_mass = src->m_mass; dst->m_ipos = src->m_ipos; dst->m_damp = src->m_damp; dst->m_fric = src->m_fric;
  dst->m_mass_dev = dst->m_mass; dst->m_ipos_dev = dst->m_ipos; dst->m_damp_dev = dst->m_damp; dst->m_fric_dev = dst->m_fric;
  dst->m_gpos = dst->m_gpos_dev = src->m_gpos; dst->m_gquat = dst->m_gquat_dev = src->m_gquat; dst->m_gsize = dst->m_gsize_dev = src->m_gsize;
  dst->hfield = src->hfield; dst->hfield_dev = src->hfield_dev; dst->timestep = dst->timestep_dev = src->timestep;
  memcpy(dst->hf_size, src->hf_size, sizeof dst->hf_size); memcpy(dst->hf_size_dev, src->hf_size_dev, sizeof dst->hf_size_dev);
  dst->m_bpos = src->m_bpos; dst->m_bpos_dev = src->m_bpos_dev;
  for (int i = 0; i < 16; i++) dst->b->radio[i] = src->b->radio[i];
  cassie_state_t *s = cassie_state_alloc(); cassie_get_state(src, s); cassie_set_state(dst, s); cassie_state_free(s);
}
cassie_sim_t *cassie_sim_duplicate(const cassie_sim_t *src) {
  cassie_sim_t *c = cassie_sim_init(src->path.c_str(), true);
  if (c) cassie_sim_copy(c, src);
  return c;
}
// batched snapshots: an opaque handle per batch (cassie_batch_state_free before cassie_batch_free)
void *cassie_batch_state_alloc(cassie_batch_t *b) { return b->impl->snap_alloc(); }
void cassie_batch_state_free(cassie_batch_t *b, void *state) { (void)b; snap_delete((Snap *)state); }
int cassie_batch_get_state(cassie_batch_t *b, void *state) { return state && b->impl->snap_get((Snap *)state) ? 0 : -1; }
int cassie_batch_set_state(cassie_batch_t *b, const void *state, const unsigned char *mask) { return state && b->impl->snap_set((const Snap *)state, mask) ? 0 : -1; }
int cassie_batch_set_reset_bank(cassie_batch_t *b, const void *state, const int *envs, int k) { return b->impl->set_reset_bank((const Snap *)state, envs, k) ? 0 : -1; }
int cassie_batch_reset_bank_size(const cassie_batch_t *b) { return b->impl->reset_bank_size(); }
int cassie_batch_reset_where(cassie_batch_t *b, const void *d_mask, const void *d_entry) { return b->impl->reset_where(d_mask, d_entry) ? 0 : -1; }
int cassie_batch_close_loops(cassie_batch_t *b, const void *d_mask, int max_iter, double tol) { return b->impl->close_loops(d_mask, max_iter, tol) ? 0 : -1; }
int cassie_batch_get_loop_status(cassie_batch_t *b, double *residual, int *iterations, double *vel_residual) { return b->impl->get_loop_status(residual, iterations, vel_residual) ? 0 : -1; }
int cassie_batch_set_ik(cassie_batch_t *b, const char *const *names, const int *kinds, const int *frames, const double *weights, int count) { return b->impl->set_ik(names, kinds, frames, weights, count) ? 0 : -1; }
int cassie_batch_solve_ik(cassie_batch_t *b, const void *d_mask, int max_iter, double tol, int velocities) { return b->impl->solve_ik(d_mask, max_iter, tol, velocities) ? 0 : -1; }
int cassie_batch_get_ik_status(cassie_batch_t *b, double *status) { return b->impl->get_ik_status(status) ? 0 : -1; }
int cassie_batch_forward_where(cassie_batch_t *b, const void *d_mask) { return b->impl->forward_where(d_mask) ? 0 : -1; }
#include "legacy_stubs.inc"
}  // extern "C"
