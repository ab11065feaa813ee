// emu_raycast.cpp -- TEST-ONLY: the product's ray source (csrc/raycast.inl) compiled with -DCASSIE_EMU on top of the host emulation of emu.cpp.  The table
// is built by the same host helper as cassie_batch_set_rays; the rows are cast for n environments that share the simulator's qpos unless the caller
// gives one per environment.  Built into its own library (tests/raycast_support.py); never linked into, loaded by, or reachable from the product library.
#include "emu.cpp"
#include "../../cassie-mujoco-sim_b200/csrc/raycast.inl"

namespace {
template <typename real> int cast_(Emu<real> &e, int n, const double *qpos, int nq, const double *genv, const float *hf, int n_terrain, const int *frame,
                                   const double *org, const double *dir, const double *maxd, int k, double *out) {
  std::vector<double> tab; std::string err;
  if (k < 1 || !ray_table(frame, org, dir, maxd, k, tab, err)) { fprintf(stderr, "emu_raycast: %s\n", err.c_str()); return -1; }
  std::vector<real> t(tab.begin(), tab.end()), q((size_t)n * QPOS_W_XB), g, rows((size_t)n * k * RAY_SLOT), ws(RS_W);
  for (int i = 0; i < n; i++) for (int c = 0; c < QPOS_W_XB; c++) q[(size_t)i * QPOS_W_XB + c] = qpos ? (c < nq ? (real)qpos[(size_t)i * nq + c] : real(0)) : e.sm[S_QPOS + c];
  if (genv) g.assign(genv, genv + (size_t)n * GEOM_ENV_W);
  const size_t cells = e.hm.nhfield ? (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0] : 0;
  RayArgs<real> A; A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = genv ? g.data() : nullptr;
  A.hfield = cells ? (hf ? hf : e.hfield.data()) : nullptr; A.n_terrain = hf ? n_terrain : 1; A.hfield_stride = cells;
  A.tab = t.data(); A.k = k; A.out = rows.data(); A.n = n;
  for (int env = 0; env < n; env++) raycast_env(A, env, ws.data());
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  return 0;
}
template <typename real> void root_(Emu<real> &e, double *out) {
  real p[3], R[9]; ray_root_pose(e.dm, e.sm.data() + S_QPOS, p, R);
  for (int c = 0; c < 3; c++) out[c] = p[c];
  for (int c = 0; c < 9; c++) out[3 + c] = R[c];
}
}  // namespace

extern "C" {
// cast k rays for n environments: qpos [n][nq] (null: the simulator's own for all), genv [n][GEOM_ENV_W] (null: the model block), hf [K][cells] (null: the
// simulator's terrain), out [n][k][RAY_SLOT]; -1 for a table the product would refuse
int emu_ray_cast(void *p, int n, const double *qpos, int nq, const double *genv, const float *hf, int n_terrain, const int *frame, const double *org,
                 const double *dir, const double *maxd, int k, double *out) {
  Handle *h = (Handle *)p;
  return h->fp32 ? cast_(h->f, n, qpos, nq, genv, hf, n_terrain, frame, org, dir, maxd, k, out) : cast_(h->d, n, qpos, nq, genv, hf, n_terrain, frame, org, dir, maxd, k, out);
}
// the root pose the ray source composes from the simulator's qpos: position [3], rotation [9] (row-major)
void emu_ray_root(void *p, double *out) { Handle *h = (Handle *)p; if (h->fp32) root_(h->f, out); else root_(h->d, out); }
// host geom id of each static collision slot (-1 past the last); returns the number of slots
int emu_ray_slots(void *p, int *geom) {
  Handle *h = (Handle *)p; const BuildInfo &info = h->fp32 ? h->f.info : h->d.info; const int ns = h->fp32 ? h->f.dm.ngeom_static : h->d.dm.ngeom_static;
  for (int k = 0; k < MGS; k++) geom[k] = -1;
  for (int g = 0; g < 256; g++) if (info.geom_dev[g] >= MG && info.geom_dev[g] < MGT) geom[info.geom_dev[g] - MG] = g;
  return ns;
}
// the static slots of the model block as a GEOM_ENV_W row (the placement every environment starts from)
void emu_ray_genv0(void *p, double *row) {
  Handle *h = (Handle *)p;
  if (h->fp32) { std::vector<float> r(GEOM_ENV_W); init_genv_row(h->f.dm, r.data()); for (int i = 0; i < GEOM_ENV_W; i++) row[i] = r[i]; }
  else init_genv_row(h->d.dm, row);
}
}
