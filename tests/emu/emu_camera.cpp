// emu_camera.cpp -- TEST-ONLY: the product's camera source (csrc/camera.inl) compiled with -DCASSIE_EMU on top of the host emulation of emu.cpp.  The
// camera is checked by the same host helper as the set verbs; the rows are rendered for n environments that share the simulator's qpos unless the
// caller gives one per environment.  Built into its own library (tests/camera_support.py); never linked into, loaded by, or reachable from the product.
#include "emu_raycast.cpp"   // emu.cpp and the ray helpers (emu_ray_slots: the static slots)
#include "../../cassie-mujoco-sim_b200/csrc/camera.inl"

namespace {
template <typename real> int render_(Emu<real> &e, int n, const double *qpos, int nq, const double *genv, const float *hf, int n_terrain, int body,
                                     const double *pos, const double *quat, double fovy, int W, int H, double zfar, double *out, double *poses) {
  double qn[4]; std::string err;
  if (body < 0 || body >= e.hm.nbody || !camera_check(pos, quat, fovy, W, H, zfar, qn, err)) { fprintf(stderr, "emu_camera: %s\n", err.c_str()); return -1; }
  std::vector<real> q((size_t)n * QPOS_W_XB), g, rows((size_t)n * W * H), ws(CS_W);
  for (int i = 0; i < n; i++) for (int c = 0; c < QPOS_W_XB; c++) q[(size_t)i * QPOS_W_XB + c] = qpos ? (c < nq ? (real)qpos[(size_t)i * nq + c] : real(0)) : e.sm[S_QPOS + c];
  if (genv) g.assign(genv, genv + (size_t)n * GEOM_ENV_W);
  const size_t cells = e.hm.nhfield ? (size_t)e.hm.hfield_nrow[0] * e.hm.hfield_ncol[0] : 0;
  CamArgs<real> A; A.model = &e.dm; A.qpos = q.data(); A.qpos_w = QPOS_W_XB; A.genv = genv ? g.data() : nullptr;
  A.hfield = cells ? (hf ? hf : e.hfield.data()) : nullptr; A.n_terrain = hf ? n_terrain : 1; A.hfield_stride = cells;
  A.body = body; A.width = W; A.height = H; A.tan_half = (real)std::tan(fovy * M_PI / 360); A.zfar = (real)zfar;
  for (int i = 0; i < 3; i++) A.pos[i] = (real)pos[i];
  for (int i = 0; i < 4; i++) A.quat[i] = (real)qn[i];
  A.out = rows.data(); A.n = n;
  for (int env = 0; env < n; env++) {
    camera_env(A, env, ws.data());
    if (poses && env == 0) {   // environment 0's staging: body poses (xpos [32][3], xquat [32][4]), camera position and rotation, moving geoms
      for (int i = 0; i < 3 * MB; i++) poses[i] = (double)ws[CS_XPOS + i];
      for (int i = 0; i < 4 * MB; i++) poses[3 * MB + i] = (double)ws[CS_XQUAT + i];
      for (int i = 0; i < 12; i++) poses[7 * MB + i] = (double)ws[CS_CAM + i];
      for (int i = 0; i < MG * GE_SLOT; i++) poses[7 * MB + 12 + i] = (double)ws[CS_MOV + i];
    }
  }
  for (size_t i = 0; i < rows.size(); i++) out[i] = (double)rows[i];
  return 0;
}
}  // namespace

extern "C" {
// render n environments: qpos [n][nq] (null: the simulator's own for all), genv [n][GEOM_ENV_W] (null: the model block), hf [K][cells] (null: the
// simulator's terrain), camera on body `body` at pos / quat, out [n][H][W]; poses (optional): environment 0's staged poses (see render_); -1 for a
// camera the product would refuse
int emu_cam_render(void *p, int n, const double *qpos, int nq, const double *genv, const float *hf, int n_terrain, int body, const double *pos,
                   const double *quat, double fovy, int W, int H, double zfar, double *out, double *poses) {
  Handle *h = (Handle *)p;
  return h->fp32 ? render_(h->f, n, qpos, nq, genv, hf, n_terrain, body, pos, quat, fovy, W, H, zfar, out, poses)
                 : render_(h->d, n, qpos, nq, genv, hf, n_terrain, body, pos, quat, fovy, W, H, zfar, out, poses);
}
// host geom id of each moving collision slot (-1 past the last); returns the number of slots
int emu_cam_moving(void *p, int *geom) {
  Handle *h = (Handle *)p; const BuildInfo &info = h->fp32 ? h->f.info : h->d.info; const int nm = h->fp32 ? h->f.dm.ngeom : h->d.dm.ngeom;
  for (int k = 0; k < MG; k++) geom[k] = -1;
  for (int g = 0; g < 256; g++) if (info.geom_dev[g] >= 0 && info.geom_dev[g] < MG) geom[info.geom_dev[g]] = g;
  return nm;
}
}
