// emu_env_body_pos.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment
// body-offset row (csrc/devmodel.h BP_W).  With the row on, a simulator runs step_env<..., F_ALL | F_BP>, the source of the F_BP kernel instances
// (extended kind), and the ray and camera sources read the row as the batch's kernels do.  Built into its own library (tests/test_env_body_pos.py);
// never linked into, loaded by, or reachable from the product library.
#include <map>
#include "emu_camera.cpp"   // emu.cpp, the ray and the camera sources

namespace {
template <typename real> struct BodyRow { real row[BP_W]; bool on = false; };
struct BodyRows { BodyRow<float> f; BodyRow<double> d; };
std::map<void *, BodyRows> g_bp;   // per simulator handle

template <typename real> void run_(Emu<real> &e, BodyRow<real> &r, int nticks, int mode) {
  if (!r.on) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.env = 0;
  step_env<real, true, F_ALL | F_BP>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.row);
}
// this environment's offsets [nbody][3] (the batch's rows are in the batch precision, the rest of the row zero)
template <typename real> void set_(Emu<real> &e, BodyRow<real> &r, const double *pos) {
  for (int i = 0; i < BP_W; i++) r.row[i] = i < 3 * e.hm.nbody ? (real)pos[i] : real(0);
  r.on = true;
}
template <typename real> void set_const_(Emu<real> &e, BodyRow<real> &r) {   // mode 3 at qpos0 with the row, as the batch's set_const launch
  e.enable_cenv();
  std::vector<real> keep(e.sm.begin() + S_QPOS, e.sm.begin() + S_QPOS + QPOS_W_XB);
  for (int i = 0; i < QPOS_W_XB; i++) e.sm[S_QPOS + i] = e.dm.qpos0[i];
  run_(e, r, 1, 3);
  for (int i = 0; i < QPOS_W_XB; i++) e.sm[S_QPOS + i] = keep[i];
}
template <typename real> int rays_(Emu<real> &e, BodyRow<real> &r, const int *frame, const double *org, const double *dir, const double *maxd, int k, double *out) {
  std::vector<double> tab; std::string err;
  if (k < 1 || !ray_table(frame, org, dir, maxd, k, tab, err)) return -1;
  std::vector<real> t(tab.begin(), tab.end()), q(e.sm.begin() + S_QPOS, e.sm.begin() + S_QPOS + QPOS_W_XB), rows((size_t)k * RAY_SLOT), ws(RS_W);
  const size_t cells = e.hm.nhfield ? (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0] : 0;
  RayArgs<real> A; A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = nullptr; A.hfield = cells ? e.hfield.data() : nullptr; A.n_terrain = 1; A.hfield_stride = cells;
  A.tab = t.data(); A.k = k; A.out = rows.data(); A.n = 1; A.bpos = r.on ? r.row : nullptr;
  raycast_env(A, 0, ws.data());
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  return 0;
}
template <typename real> int cam_(Emu<real> &e, BodyRow<real> &r, int body, const double *pos, const double *quat, double fovy, int W, int H, double zfar, double *out) {
  double qn[4]; std::string err;
  if (body < 0 || body >= e.hm.nbody || !camera_check(pos, quat, fovy, W, H, zfar, qn, err)) return -1;
  std::vector<real> q(e.sm.begin() + S_QPOS, e.sm.begin() + S_QPOS + QPOS_W_XB), rows((size_t)W * H), ws(CS_W);
  const size_t cells = e.hm.nhfield ? (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0] : 0;
  CamArgs<real> A; A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = nullptr; A.hfield = cells ? e.hfield.data() : nullptr; A.n_terrain = 1; A.hfield_stride = cells;
  A.body = body; A.width = W; A.height = H; A.tan_half = (real)std::tan(fovy * M_PI / 360); A.zfar = (real)zfar;
  for (int i = 0; i < 3; i++) A.pos[i] = (real)pos[i];
  for (int i = 0; i < 4; i++) A.quat[i] = (real)qn[i];
  A.out = rows.data(); A.n = 1; A.bpos = r.on ? r.row : nullptr;
  camera_env(A, 0, ws.data());
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  return 0;
}
}  // namespace

extern "C" {
void *emu_bp_new(const char *path, int fp32) { void *p = emu_new(path, fp32); if (p) g_bp.erase(p); return p; }
void emu_bp_free(void *p) { g_bp.erase(p); emu_free(p); }
void emu_bp_set(void *p, const double *pos) { Handle *h = (Handle *)p; BodyRows &r = g_bp[p]; if (h->fp32) set_(h->f, r.f, pos); else set_(h->d, r.d, pos); }
void emu_bp_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; BodyRows &r = g_bp[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, r.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, r.d, nticks, 0); }
}
void emu_bp_forward(void *p) { Handle *h = (Handle *)p; BodyRows &r = g_bp[p]; if (h->fp32) run_(h->f, r.f, 1, 1); else run_(h->d, r.d, 1, 1); }
void emu_bp_set_const(void *p) { Handle *h = (Handle *)p; BodyRows &r = g_bp[p]; if (h->fp32) set_const_(h->f, r.f); else set_const_(h->d, r.d); }
int emu_bp_rays(void *p, const int *frame, const double *org, const double *dir, const double *maxd, int k, double *out) {
  Handle *h = (Handle *)p; BodyRows &r = g_bp[p]; return h->fp32 ? rays_(h->f, r.f, frame, org, dir, maxd, k, out) : rays_(h->d, r.d, frame, org, dir, maxd, k, out); }
int emu_bp_camera(void *p, int body, const double *pos, const double *quat, double fovy, int W, int H, double zfar, double *out) {
  Handle *h = (Handle *)p; BodyRows &r = g_bp[p]; return h->fp32 ? cam_(h->f, r.f, body, pos, quat, fovy, W, H, zfar, out) : cam_(h->d, r.d, body, pos, quat, fovy, W, H, zfar, out); }
// the model's offsets into the simulator's own block (the shared placement; the oracle's and the legacy verbs' semantics) -- the row is left alone
int emu_bp_set_model(void *p, const double *pos) {
  Handle *h = (Handle *)p; std::string err;
  if (h->fp32) { for (int i = 0; i < 3 * h->f.hm.nbody; i++) h->f.hm.body_pos[i] = pos[i]; return build_dev_model(h->f.hm, h->f.dm, err, &h->f.info) ? 0 : -1; }
  for (int i = 0; i < 3 * h->d.hm.nbody; i++) h->d.hm.body_pos[i] = pos[i]; return build_dev_model(h->d.hm, h->d.dm, err, &h->d.info) ? 0 : -1;
}
// the broad phase's robot bound: the block's, and robot_reach_of's for offsets pos (with build_dev_model's slack, in the batch precision)
void emu_bp_reach(void *p, const double *pos, double *out2) {
  Handle *h = (Handle *)p;
  if (h->fp32) { out2[0] = h->f.dm.robot_reach; out2[1] = (float)(robot_reach_of(h->f.hm, pos, h->f.dm.root_body, h->f.dm.xb, h->f.info.geom_dev) * 1.05 + 0.05); }
  else { out2[0] = h->d.dm.robot_reach; out2[1] = robot_reach_of(h->d.hm, pos, h->d.dm.root_body, h->d.dm.xb, h->d.info.geom_dev) * 1.05 + 0.05; }
}
// the verb's refusal rule for body b: 0 changeable, 1 not (world, welded to the world, extra free body)
int emu_bp_refused(void *p, int b) { Handle *h = (Handle *)p; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm; return env_body_pos_check(m, b, h->fp32 ? h->f.dm.xb : h->d.dm.xb).empty() ? 0 : 1; }
}
