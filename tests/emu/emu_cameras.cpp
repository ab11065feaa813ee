// emu_cameras.cpp -- TEST-ONLY: the product's camera-set source (csrc/camera_set.inl) compiled with -DCASSIE_EMU on top of the host emulation of
// emu.cpp: k cameras in one pass, per-environment mount rows and geom-id rows.  The mounts are checked and prepared as the batch's set verb and
// render do (csrc/cassie_b200.cu); the geom table is the batch's device-to-model one.  Built into its own library (tests/camera_set_support.py); never
// linked into, loaded by, or reachable from the product.
#include "emu_raycast.cpp"   // emu.cpp and the ray helpers (emu_ray_slots: the static slots)
#include "../../cassie-mujoco-sim_b200/csrc/camera_set.inl"

namespace {
template <typename real> int renders_(Emu<real> &e, int n, const double *qpos, int nq, const double *genv, const float *hf, int n_terrain, int k,
                                      const int *body, const double *pos, const double *quat, const double *fovy, int W, int H, double zfar,
                                      const double *cenv, double *out, int *geom) {
  if (k < 1 || k > CAM_MAX) return -1;
  CamSetArgs<real> A{}; std::string err;
  std::vector<real> q((size_t)n * QPOS_W_XB), g, ce, rows((size_t)n * k * W * H), ws(CSET_W);
  std::vector<int> gid(geom ? rows.size() : 0), tab(MGT, -1);
  for (int c = 0; c < k; c++) {
    double qn[4];
    if (body[c] < 0 || body[c] >= e.hm.nbody || !camera_check(pos + 3 * c, quat + 4 * c, fovy[c], W, H, zfar, qn, err)) { fprintf(stderr, "emu_cameras: %s\n", err.c_str()); return -1; }
    CamMount<real> &m = A.cam[c]; m.body = body[c]; m.tan_half = (real)std::tan(fovy[c] * M_PI / 360);
    for (int i = 0; i < 3; i++) m.pos[i] = (real)pos[3 * c + i];
    for (int i = 0; i < 4; i++) m.quat[i] = (real)qn[i];
  }
  for (int i = 0; i < n; i++) for (int c = 0; c < QPOS_W_XB; c++) q[(size_t)i * QPOS_W_XB + c] = qpos ? (c < nq ? (real)qpos[(size_t)i * nq + c] : real(0)) : e.sm[S_QPOS + c];
  if (genv) g.assign(genv, genv + (size_t)n * GEOM_ENV_W);
  if (cenv) ce.assign(cenv, cenv + (size_t)n * k * CAMENV_SLOT);
  for (int h = 0; h < e.hm.ngeom && h < 256; h++) if (e.info.geom_dev[h] >= 0 && e.info.geom_dev[h] < MGT) tab[e.info.geom_dev[h]] = h;
  const size_t cells = e.hm.nhfield ? (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0] : 0;
  A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = genv ? g.data() : nullptr;
  A.hfield = cells ? (hf ? hf : e.hfield.data()) : nullptr; A.n_terrain = hf ? n_terrain : 1; A.hfield_stride = cells;
  A.width = W; A.height = H; A.zfar = (real)zfar; A.k = k;
  A.cenv = cenv ? ce.data() : nullptr; A.geom = geom ? gid.data() : nullptr; A.gtab = tab.data();
  A.out = rows.data(); A.n = n;
  for (int env = 0; env < n; env++) camera_set_env(A, env, ws.data());
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  if (geom) for (size_t i = 0; i < gid.size(); i++) geom[i] = gid[i];
  return 0;
}
}  // namespace

extern "C" {
// render n environments with k cameras in one pass: qpos [n][nq] (null: the simulator's own for all), genv [n][GEOM_ENV_W] (null: the model block),
// hf [K][cells] (null: the simulator's terrain), cameras body [k], pos [k][3], quat [k][4], fovy [k]; cenv [n][k][CAMENV_SLOT] per-environment mount
// rows (null: none; cast to the precision as the device rows hold them); out [n][k][H][W]; geom [n][k][H][W] model geom ids (null: none); -1 for a set
// the product would refuse
int emu_cams_render(void *p, int n, const double *qpos, int nq, const double *genv, const float *hf, int n_terrain, int k, const int *body,
                    const double *pos, const double *quat, const double *fovy, int W, int H, double zfar, const double *cenv, double *out, int *geom) {
  Handle *h = (Handle *)p;
  return h->fp32 ? renders_(h->f, n, qpos, nq, genv, hf, n_terrain, k, body, pos, quat, fovy, W, H, zfar, cenv, out, geom)
                 : renders_(h->d, n, qpos, nq, genv, hf, n_terrain, k, body, pos, quat, fovy, W, H, zfar, cenv, out, geom);
}
}
