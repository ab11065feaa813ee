// emu_loops.cpp -- TEST-ONLY: the product's loop-closure source (csrc/loops.inl) compiled with -DCASSIE_EMU on top of the host emulation of emu.cpp.  The
// table is built by the same host helper as cassie_batch_close_loops, and every environment runs the kernel's per-warp body with its phases as loops over
// 32 lanes.  Built into its own library (tests/test_close_loops.py); never linked into, loaded by, or reachable from the product library.
#include "emu.cpp"
#include "../../cassie-mujoco-sim_b200/csrc/loops.inl"

namespace {
template <typename real> int close_(Emu<real> &e, int n, double *qpos, double *qvel, const unsigned char *mask, const double *bpos, int max_iter, double tol,
                                    double *status) {
  LoopArgs<real> A; std::string err;
  if (!loop_table(e.hm, A.T, err)) { fprintf(stderr, "emu_loops: %s\n", err.c_str()); return -1; }
  const int nq = e.hm.nq, nv = e.hm.nv, qw = e.dm.qpos_w, vw = e.dm.qvel_w, nb = e.hm.nbody;
  std::vector<real> q((size_t)n * qw, real(0)), v((size_t)n * vw, real(0)), bp, st((size_t)n * LOOP_SLOT, real(0)), ws(LW_SIZE);
  for (int i = 0; i < n; i++) {
    for (int c = 0; c < nq; c++) q[(size_t)i * qw + c] = (real)qpos[(size_t)i * nq + c];
    for (int c = 0; c < nv; c++) v[(size_t)i * vw + c] = (real)qvel[(size_t)i * nv + c];
    for (int c = 0; c < LOOP_SLOT; c++) st[(size_t)i * LOOP_SLOT + c] = (real)status[(size_t)i * LOOP_SLOT + c];
  }
  if (bpos) { bp.assign((size_t)n * BP_W, real(0)); for (int i = 0; i < n; i++) for (int c = 0; c < 3 * nb; c++) bp[(size_t)i * BP_W + c] = (real)bpos[(size_t)i * 3 * nb + c]; }
  A.model = &e.dm; A.qpos = q.data(); A.qpos_w = qw; A.qvel = v.data(); A.qvel_w = vw; A.bpos = bpos ? bp.data() : nullptr; A.status = st.data();
  A.mask = mask; A.n = n; A.max_iter = max_iter; A.tol = (real)tol;
  int count = 0;
  if (A.T.nrow) for (int env = 0; env < n; env++) count += loops_env(A, env, ws.data()) ? 1 : 0;
  for (int i = 0; i < n; i++) {
    for (int c = 0; c < nq; c++) qpos[(size_t)i * nq + c] = (double)q[(size_t)i * qw + c];
    for (int c = 0; c < nv; c++) qvel[(size_t)i * nv + c] = (double)v[(size_t)i * vw + c];
    for (int c = 0; c < LOOP_SLOT; c++) status[(size_t)i * LOOP_SLOT + c] = (double)st[(size_t)i * LOOP_SLOT + c];
  }
  return count;
}
}  // namespace

extern "C" {
// close the loops of n environments in place: qpos [n][nq], qvel [n][nv], status [n][LOOP_SLOT] (rows of unselected environments are kept), mask [n]
// (null: all), bpos [n][nbody][3] body offsets (null: the model's).  Returns the number of environments selected, or -1 for a model the product refuses
int emu_close_loops(void *p, int n, double *qpos, double *qvel, const unsigned char *mask, const double *bpos, int max_iter, double tol, double *status) {
  Handle *h = (Handle *)p;
  return h->fp32 ? close_(h->f, n, qpos, qvel, mask, bpos, max_iter, tol, status) : close_(h->d, n, qpos, qvel, mask, bpos, max_iter, tol, status);
}
// the free coordinates of the model: qpos addresses [nq] flags (1: free) and dof flags [nv]; returns the number of free dofs, or -1
int emu_loop_free(void *p, int *qfree, int *vfree) {
  Handle *h = (Handle *)p; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm;
  LoopTable T; std::string err;
  if (!loop_table(m, T, err)) return -1;
  for (int i = 0; i < m.nq; i++) qfree[i] = 0;
  for (int i = 0; i < m.nv; i++) vfree[i] = 0;
  for (int i = 0; i < T.nfj; i++) { const int j = T.fj_jnt[i]; for (int c = 0; c < (m.jnt_type[j] == JNT_BALL ? 4 : 1); c++) qfree[m.jnt_qposadr[j] + c] = 1; }
  for (int k = 0; k < T.nf; k++) vfree[T.fdof[k]] = 1;
  return T.nf;
}
}
