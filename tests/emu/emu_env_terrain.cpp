// emu_env_terrain.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a bank of terrains, a
// per-environment static-geom row (csrc/devmodel.h GEOM_ENV_W) and a terrain selection, as a batch with per-environment terrain holds them.  The
// simulator stands for environment `env` of such a batch and runs step_env<..., F_ALL | F_EG | F_TR>, the source of the F_TR kernel instances (or the
// F_EG source with the same row, or the plain F_ALL source), with the bank entry chosen as the kernel wrapper chooses it.  The row's height-field slot
// is filled by the same host helper as cassie_batch_set_env_hfield.  The ray and camera sources (csrc/raycast.inl, camera.inl) are cast here with a
// selection row too.  Built into its own library (tests/test_env_terrain.py); never linked into, loaded by, or reachable from the product library.
#include <map>
#include "emu_camera.cpp"   // emu.cpp, the ray source and the camera source

namespace {
template <typename real> struct TerrainState { real row[GEOM_ENV_W]; int mode = 0, env = 0, terrain = 0; };   // mode 0 plain F_ALL, 1 F_EG, 2 F_EG | F_TR
struct TerrainStates { TerrainState<float> f; TerrainState<double> d; std::vector<float> bank; int K = 1; };
std::map<void *, TerrainStates> g_tr;   // per simulator handle

template <typename real> void run_(Emu<real> &e, TerrainStates &S, TerrainState<real> &r, int nticks, int mode) {
  const size_t cells = (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0];
  EnvPtrs<real> E = e.ptrs(); E.genv = r.row; E.env = 0;   // the row is this environment's
  if (!S.bank.empty()) E.hfield = S.bank.data() + (size_t)(r.env % S.K) * cells;   // the wrapper's default: environment env stands on entry env % K
  if (r.mode == 2 && !S.bank.empty()) E.hfield = S.bank.data() + (size_t)((unsigned)r.terrain % (unsigned)S.K) * cells;   // ... F_TR: its selection
  const bool ext = e.use_cenv || e.use_ext;
  if (r.mode == 0) e.run(nticks, mode);
  else if (r.mode == 1) { if (ext) step_env<real, true, F_ALL | F_EG>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
                          else step_env<real, false, F_ALL | F_EG>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode); }
  else { if (ext) step_env<real, true, F_ALL | F_EG | F_TR>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
         else step_env<real, false, F_ALL | F_EG | F_TR>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode); }
}
// the row of a batch with per-environment terrain: the model block's placement, the height field's slot at pos / size (NULL: the shared ones)
template <typename real> void terrain_row(const Emu<real> &e, const double *pos, const double *size, real *row) {
  init_genv_row(e.dm, row);
  const int g = hfield_geom(e.hm);
  if (g < 0) return;
  env_hfield_slot(e.hm, g, pos ? pos : &e.hm.geom_pos[3 * g], size ? size : e.hm.hfield_size.data(), row + GE_SLOT * (e.info.geom_dev[g] - MG));
}
template <typename real> int set_(Emu<real> &e, TerrainState<real> &r, int mode, int env, int terrain, const double *pos, const double *size) {
  if (size && !hfield_size_check(size).empty()) return -1;
  r.mode = mode; r.env = env; r.terrain = terrain;
  terrain_row(e, pos, size, r.row);
  if (mode == 1) init_genv_row(e.dm, r.row);   // F_EG: the row a batch without terrain rows carries
  return 0;
}
template <typename real> int cast_tr_(Emu<real> &e, const TerrainStates &S, int n, const double *qpos, int nq, const double *genv, const int *terrain, const int *frame,
                                      const double *org, const double *dir, const double *maxd, int k, double *out) {
  std::vector<double> tab; std::string err;
  if (k < 1 || !ray_table(frame, org, dir, maxd, k, tab, err)) return -1;
  std::vector<real> t(tab.begin(), tab.end()), q((size_t)n * QPOS_W_XB), g(genv, genv + (size_t)n * GEOM_ENV_W), rows((size_t)n * k * RAY_SLOT), ws(RS_W);
  for (int i = 0; i < n; i++) for (int c = 0; c < QPOS_W_XB; c++) q[(size_t)i * QPOS_W_XB + c] = c < nq ? (real)qpos[(size_t)i * nq + c] : real(0);
  RayArgs<real> A; A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = g.data();
  A.hfield = S.bank.data(); A.n_terrain = S.K; A.hfield_stride = (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0]; A.terrain = terrain;
  A.tab = t.data(); A.k = k; A.out = rows.data(); A.n = n;
  for (int env = 0; env < n; env++) raycast_env(A, env, ws.data());
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  return 0;
}
template <typename real> int render_tr_(Emu<real> &e, const TerrainStates &S, int n, const double *qpos, int nq, const double *genv, const int *terrain, int body,
                                        const double *pos, const double *quat, double fovy, int W, int H, double zfar, double *out) {
  double qn[4]; std::string err;
  if (body < 0 || body >= e.hm.nbody || !camera_check(pos, quat, fovy, W, H, zfar, qn, err)) return -1;
  std::vector<real> q((size_t)n * QPOS_W_XB), g(genv, genv + (size_t)n * GEOM_ENV_W), rows((size_t)n * W * H), ws(CS_W);
  for (int i = 0; i < n; i++) for (int c = 0; c < QPOS_W_XB; c++) q[(size_t)i * QPOS_W_XB + c] = c < nq ? (real)qpos[(size_t)i * nq + c] : real(0);
  CamArgs<real> A; A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = g.data();
  A.hfield = S.bank.data(); A.n_terrain = S.K; A.hfield_stride = (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0]; A.terrain = terrain;
  A.body = body; A.width = W; A.height = H; A.tan_half = (real)std::tan(fovy * M_PI / 360); A.zfar = (real)zfar;
  for (int i = 0; i < 3; i++) A.pos[i] = (real)pos[i];
  for (int i = 0; i < 4; i++) A.quat[i] = (real)qn[i];
  A.out = rows.data(); A.n = n;
  for (int env = 0; env < n; env++) camera_env(A, env, ws.data());
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  return 0;
}
}  // namespace

extern "C" {
void *emu_tr_new(const char *path, int fp32) { void *p = emu_new(path, fp32); if (p) g_tr.erase(p); return p; }
void emu_tr_free(void *p) { g_tr.erase(p); emu_free(p); }
// the bank: K terrains of nrow * ncol normalised elevations
void emu_tr_bank(void *p, const float *data, int K) {
  Handle *h = (Handle *)p; TerrainStates &S = g_tr[p]; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm;
  S.K = K; S.bank.assign(data, data + (size_t)K * m.hfield_nrow[0] * m.hfield_ncol[0]);
}
// this simulator is environment `env` of a batch: mode 0 plain (no row), 1 the F_EG row of a batch without terrain rows, 2 per-environment terrain with
// selection `terrain` and the height field at pos / size (NULL: the shared ones); -1 for a size the verb refuses
int emu_tr_set(void *p, int mode, int env, int terrain, const double *pos, const double *size) {
  Handle *h = (Handle *)p; TerrainStates &S = g_tr[p];
  return h->fp32 ? set_(h->f, S.f, mode, env, terrain, pos, size) : set_(h->d, S.d, mode, env, terrain, pos, size);
}
void emu_tr_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; TerrainStates &S = g_tr[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, S, S.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, S, S.d, nticks, 0); }
}
void emu_tr_forward(void *p) { Handle *h = (Handle *)p; TerrainStates &S = g_tr[p]; if (h->fp32) run_(h->f, S, S.f, 1, 1); else run_(h->d, S, S.d, 1, 1); }
// a GEOM_ENV_W row with the height field's slot at pos / size (NULL: shared), as cassie_batch_set_env_hfield writes it
void emu_tr_row(void *p, const double *pos, const double *size, double *out) {
  Handle *h = (Handle *)p;
  if (h->fp32) { float r[GEOM_ENV_W]; terrain_row(h->f, pos, size, r); for (int i = 0; i < GEOM_ENV_W; i++) out[i] = r[i]; }
  else terrain_row(h->d, pos, size, out);
}
// rays / depth images for n environments with rows genv [n][GEOM_ENV_W], the bank of emu_tr_bank and selections terrain [n] (NULL: e % K)
int emu_tr_ray_cast(void *p, int n, const double *qpos, int nq, const double *genv, const int *terrain, const int *frame, const double *org, const double *dir,
                    const double *maxd, int k, double *out) {
  Handle *h = (Handle *)p; const TerrainStates &S = g_tr[p];
  return h->fp32 ? cast_tr_(h->f, S, n, qpos, nq, genv, terrain, frame, org, dir, maxd, k, out) : cast_tr_(h->d, S, n, qpos, nq, genv, terrain, frame, org, dir, maxd, k, out);
}
int emu_tr_render(void *p, int n, const double *qpos, int nq, const double *genv, const int *terrain, int body, const double *pos, const double *quat, double fovy,
                  int W, int H, double zfar, double *out) {
  Handle *h = (Handle *)p; const TerrainStates &S = g_tr[p];
  return h->fp32 ? render_tr_(h->f, S, n, qpos, nq, genv, terrain, body, pos, quat, fovy, W, H, zfar, out)
                 : render_tr_(h->d, S, n, qpos, nq, genv, terrain, body, pos, quat, fovy, W, H, zfar, out);
}
}
