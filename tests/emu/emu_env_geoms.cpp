// emu_env_geoms.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment
// static-geom row (csrc/devmodel.h GEOM_ENV_W).  With the row on, a simulator runs step_env<..., F_ALL | F_EG>, the source of the F_EG kernel
// instances, and the row is filled by the same host helpers as cassie_batch_set_env_geom_pose.  Built into its own library (tests/test_env_geoms.py);
// never linked into, loaded by, or reachable from the product library.
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct GeomRow { real row[GEOM_ENV_W]; bool on = false; };
struct GeomRows { GeomRow<float> f; GeomRow<double> d; };
std::map<void *, GeomRows> g_rows;   // per simulator handle

template <typename real> void run_(Emu<real> &e, GeomRow<real> &r, int nticks, int mode) {
  if (!r.on) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.genv = r.row; E.env = 0;
  if (e.use_cenv || e.use_ext) step_env<real, true, F_ALL | F_EG>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
  else step_env<real, false, F_ALL | F_EG>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
}
template <typename real> void enable_(Emu<real> &e, GeomRow<real> &r) { if (!r.on) { init_genv_row(e.dm, r.row); r.on = true; } }
// this environment's placement of host geom g (NULL parts: the model's)
template <typename real> int set_(Emu<real> &e, GeomRow<real> &r, int g, const double *pos, const double *quat, const double *size) {
  std::string err; const int k = env_geom_check(e.hm, e.info.geom_dev, g, err);
  if (k < 0) return -1;
  enable_(e, r);
  env_geom_slot(e.hm, g, pos ? pos : &e.hm.geom_pos[3 * g], quat ? quat : &e.hm.geom_quat[4 * g], size ? size : &e.hm.geom_size[3 * g], r.row + GE_SLOT * k);
  return 0;
}
}  // namespace

extern "C" {
void *emu_eg_new(const char *path, int fp32) { void *p = emu_new(path, fp32); if (p) g_rows.erase(p); return p; }
void emu_eg_free(void *p) { g_rows.erase(p); emu_free(p); }
void emu_eg_enable(void *p) { Handle *h = (Handle *)p; GeomRows &r = g_rows[p]; if (h->fp32) enable_(h->f, r.f); else enable_(h->d, r.d); }
int emu_eg_set(void *p, int g, const double *pos, const double *quat, const double *size) {
  Handle *h = (Handle *)p; GeomRows &r = g_rows[p]; return h->fp32 ? set_(h->f, r.f, g, pos, quat, size) : set_(h->d, r.d, g, pos, quat, size); }
void emu_eg_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; GeomRows &r = g_rows[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, r.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, r.d, nticks, 0); }
}
void emu_eg_forward(void *p) { Handle *h = (Handle *)p; GeomRows &r = g_rows[p]; if (h->fp32) run_(h->f, r.f, 1, 1); else run_(h->d, r.d, 1, 1); }
// the row [GEOM_ENV_W] (zeros while off), the model block's static poses [MGS][12], a host geom's collision slot (-1: none), and the world pose [12]
// the factored host helper composes for a static geom's model placement
void emu_eg_row(void *p, double *out) { Handle *h = (Handle *)p; GeomRows &r = g_rows[p]; for (int i = 0; i < GEOM_ENV_W; i++) out[i] = h->fp32 ? (r.f.on ? r.f.row[i] : 0) : (r.d.on ? r.d.row[i] : 0); }
void emu_eg_block_wpose(void *p, double *out) { Handle *h = (Handle *)p; for (int k = 0; k < MGS; k++) for (int c = 0; c < 12; c++) out[12 * k + c] = h->fp32 ? h->f.dm.geom_wpose[k][c] : h->d.dm.geom_wpose[k][c]; }
int emu_eg_geom_slot(void *p, int g) { Handle *h = (Handle *)p; const BuildInfo &i = h->fp32 ? h->f.info : h->d.info; return g >= 0 && g < 256 ? i.geom_dev[g] : -1; }
void emu_eg_static_wpose(void *p, int g, double *out12) { Handle *h = (Handle *)p; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm; static_geom_wpose(m, g, &m.geom_pos[3 * g], &m.geom_quat[4 * g], out12); }
}
