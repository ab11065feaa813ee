// emu_ik.cpp -- TEST-ONLY: the product's inverse-kinematics source (csrc/ik.inl) compiled with -DCASSIE_EMU on top of the host emulation of emu.cpp.  The
// table is built by the same host helper as cassie_batch_set_ik, and every environment runs the kernel's per-warp body with its phases as loops over 32
// lanes.  Built into its own library (tests/ik_support.py); never linked into, loaded by, or reachable from the product library.
#include "emu.cpp"
#include "../../cassie-mujoco-sim_b200/csrc/ik.inl"

namespace {
template <typename real> int solve_(Emu<real> &e, int n, double *qpos, double *qvel, const unsigned char *mask, const double *bpos, int nt, const int *body,
                                    const int *frame, const double *fpos, const double *fquat, const double *w, const double *targets, int max_iter,
                                    double tol, double loop_tol, int velocities, double *status) {
  IkArgs<real> A; std::string err;
  if (!ik_table<real>(e.hm, nt, body, frame, fpos, fquat, w, A.I, err)) { fprintf(stderr, "emu_ik: %s\n", err.c_str()); return -1; }
  const int nq = e.hm.nq, nv = e.hm.nv, qw = e.dm.qpos_w, vw = e.dm.qvel_w, nb = e.hm.nbody;
  std::vector<real> q((size_t)n * qw, real(0)), v((size_t)n * vw, real(0)), bp, tg((size_t)n * IK_MAX * IK_TW), st((size_t)n * IK_SLOT, real(0)), ws(IW_SIZE);
  for (int i = 0; i < n; i++) {
    for (int c = 0; c < nq; c++) q[(size_t)i * qw + c] = (real)qpos[(size_t)i * nq + c];
    for (int c = 0; c < nv; c++) v[(size_t)i * vw + c] = (real)qvel[(size_t)i * nv + c];
    for (int c = 0; c < IK_SLOT; c++) st[(size_t)i * IK_SLOT + c] = (real)status[(size_t)i * IK_SLOT + c];
  }
  for (size_t i = 0; i < tg.size(); i++) tg[i] = (real)targets[i];
  if (bpos) { bp.assign((size_t)n * BP_W, real(0)); for (int i = 0; i < n; i++) for (int c = 0; c < 3 * nb; c++) bp[(size_t)i * BP_W + c] = (real)bpos[(size_t)i * 3 * nb + c]; }
  A.model = &e.dm; A.qpos = q.data(); A.qpos_w = qw; A.qvel = v.data(); A.qvel_w = vw; A.bpos = bpos ? bp.data() : nullptr; A.targets = tg.data();
  A.status = st.data(); A.mask = mask; A.n = n; A.max_iter = max_iter; A.velocities = velocities; A.tol = (real)tol; A.loop_tol = (real)loop_tol;
  int count = 0;
  for (int env = 0; env < n; env++) count += ik_env(A, env, ws.data()) ? 1 : 0;
  for (int i = 0; i < n; i++) {
    for (int c = 0; c < nq; c++) qpos[(size_t)i * nq + c] = (double)q[(size_t)i * qw + c];
    for (int c = 0; c < nv; c++) qvel[(size_t)i * nv + c] = (double)v[(size_t)i * vw + c];
    for (int c = 0; c < IK_SLOT; c++) status[(size_t)i * IK_SLOT + c] = (double)st[(size_t)i * IK_SLOT + c];
  }
  return count;
}
}  // namespace

extern "C" {
// solve n environments in place: qpos [n][nq], qvel [n][nv], status [n][IK_SLOT] (rows of unselected environments are kept), mask [n] (null: all), bpos
// [n][nbody][3] (null: the model's); nt targets: body ids, frames (0 world, 1 root), the frame in its body fpos [nt][3] / fquat [nt][4], weights [nt][6];
// target rows [n][IK_MAX][IK_TW].  Returns the number of environments selected, or -1 for a target list the product refuses
int emu_solve_ik(void *p, int n, double *qpos, double *qvel, const unsigned char *mask, const double *bpos, int nt, const int *body, const int *frame,
                 const double *fpos, const double *fquat, const double *w, const double *targets, int max_iter, double tol, double loop_tol, int velocities,
                 double *status) {
  Handle *h = (Handle *)p;
  return h->fp32 ? solve_(h->f, n, qpos, qvel, mask, bpos, nt, body, frame, fpos, fquat, w, targets, max_iter, tol, loop_tol, velocities, status)
                 : solve_(h->d, n, qpos, qvel, mask, bpos, nt, body, frame, fpos, fquat, w, targets, max_iter, tol, loop_tol, velocities, status);
}
// the free columns of the solve: their dofs [nv] flags (1: free) and, per column, its dof, limited flag and range; returns the column count, or -1
int emu_ik_columns(void *p, int *dof, int *lim, double *lo, double *hi) {
  Handle *h = (Handle *)p; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm;
  IkTable<double> I; std::string err;
  if (!ik_table<double>(m, 0, nullptr, nullptr, nullptr, nullptr, nullptr, I, err)) return -1;
  for (int c = 0; c < I.F.nf; c++) { dof[c] = I.F.fdof[c]; lim[c] = I.col_lim[c]; lo[c] = I.col_lo[c]; hi[c] = I.col_hi[c]; }
  return I.F.nf;
}
}
