// emu_contacts.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) with the contact lists of the
// F_CL instances.  A simulator runs the contact-list twin's source, step_env<..., F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF | F_CL>, with the
// offset, actuator, mechanics and contact rows holding the model's values and zero applied forces (what a batch with contact lists carries there), an
// optional frame table and a contact-list row [CON_W]; or, unlisted, the chain twin's source (the same without F_CL) on the same rows.  The aux row
// stays as emu.cpp has it (on).  Built into its own library (tests/test_contacts.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <map>
#include "emu.cpp"

namespace {
constexpr int CHAIN = F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF;
template <typename real> struct ClRows {
  real bp[BP_W], act[ACT_W], mech[MECH_W], ct[CONTACT_W], app[APPLIED_W], row[CON_W];
  int geom[MGT];
  std::vector<real> ftab, frames; int nfr = 0; bool listed = true;
};
struct ClSim { ClRows<float> f; ClRows<double> d; };
std::map<void *, ClSim> g_cl;   // per simulator handle

template <typename real> void run_(Emu<real> &e, ClRows<real> &r, int nticks, int mode) {
  EnvPtrs<real> E = e.ptrs(); E.env = 0; E.genv = nullptr; E.jac = nullptr; E.jfr = 0;
  E.ftab = r.nfr ? r.ftab.data() : nullptr; E.frames = r.nfr ? r.frames.data() : nullptr; E.nfr = r.nfr;
  if (r.listed) {
    const ContactListArgs<real> cl{r.row, r.geom};
    step_env<real, true, CHAIN | F_CL>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app, TraceArgs<real>{}, cl);
  } else {
    step_env<real, true, CHAIN>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app);
  }
}
template <typename real> int slot_(const Emu<real> &e, int g) { return g < 256 && e.info.geom_dev[g] >= 0 && e.info.geom_dev[g] < MGT ? e.info.geom_dev[g] : -1; }
// the model's offsets, actuators, mechanics and contact softness in the rows, zero applied forces (as emu_trace.cpp), and the geom table as
// cassie_batch_enable_contacts builds it
template <typename real> void init_(Emu<real> &e, ClRows<real> &r) {
  const HostModel &m = e.hm;
  for (int i = 0; i < BP_W; i++) r.bp[i] = i < 3 * m.nbody ? (real)m.body_pos[i] : real(0);
  for (int i = 0; i < ACT_W; i++) r.act[i] = 0;
  for (int i = 0; i < m.nu && i < MU; i++) {
    r.act[AC_LO + i] = e.dm.act_ctrl_lo[i]; r.act[AC_HI + i] = e.dm.act_ctrl_hi[i];
    r.act[AC_WMAX + i] = (real)(m.actuator_user[i] * 2 * M_PI / 60); r.act[AC_DELAY + i] = AC_MAXDELAY;
  }
  for (int i = 0; i < MECH_W; i++) r.mech[i] = 0;
  for (int i = 0; i < 3 * m.nbody; i++) r.mech[MC_INERTIA + i] = (real)m.body_inertia[i];
  for (int i = 0; i < e.dm.nv; i++) {
    const int j = m.dof_jntid[i];
    r.mech[MC_ARMATURE + i] = (real)m.dof_armature[i]; r.mech[MC_STIFF + i] = (real)m.jnt_stiffness[j]; r.mech[MC_SPRING + i] = (real)m.qpos_spring[m.jnt_qposadr[j]];
  }
  for (int i = 0; i < CONTACT_W; i++) r.ct[i] = 0;
  for (int k = 0; k < MGT; k++) r.geom[k] = -1;
  for (int g = 0; g < m.ngeom; g++) {
    const int s = slot_(e, g); if (s < 0) continue;
    r.geom[s] = g;
    real *q = r.ct + CT_SLOT * s;
    for (int k = 0; k < 2; k++) q[CT_SOLREF + k] = (real)m.geom_solref[2 * g + k];
    for (int k = 0; k < 5; k++) q[CT_SOLIMP + k] = (real)m.geom_solimp[5 * g + k];
    q[CT_SOLMIX] = (real)m.geom_solmix[g];
  }
  for (int i = 0; i < APPLIED_W; i++) r.app[i] = 0;
  for (int i = 0; i < CON_W; i++) r.row[i] = 0;
}
template <typename real> int frames_(Emu<real> &e, ClRows<real> &r, const char *const *names, const int *kinds, int count) {
  if (count < 0 || count > FRAME_MAX) return -1;
  std::vector<real> tab((size_t)count * FT_W);
  for (int f = 0; f < count; f++) { std::string err; if (frame_table_row(e.hm, names[f], kinds[f], &tab[(size_t)f * FT_W], err) < 0) return -1; }
  r.ftab = tab; r.frames.assign((size_t)count * FRAME_W, real(0)); r.nfr = count;
  return 0;
}
template <typename real> int rows_set_(Emu<real> &e, ClRows<real> &r, const std::string &what, const double *v, int n) {
  real *dst = what == "bp" ? r.bp : what == "ct" ? r.ct : nullptr; const int w = what == "bp" ? BP_W : CONTACT_W;
  if (!dst || n > w) return -1;
  for (int i = 0; i < n; i++) dst[i] = (real)v[i];
  (void)e; return 0;
}
}  // namespace

extern "C" {
void *emu_cl_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; ClSim &s = g_cl[p]; s = ClSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_cl_free(void *p) { g_cl.erase(p); emu_free(p); }
int emu_cl_set_frames(void *p, const char *const *names, const int *kinds, int count) {
  Handle *h = (Handle *)p; ClSim &s = g_cl[p]; return h->fp32 ? frames_(h->f, s.f, names, kinds, count) : frames_(h->d, s.d, names, kinds, count); }
// listed = 0 runs the chain twin's source instead (the same rows, no F_CL)
void emu_cl_listed(void *p, int on) { ClSim &s = g_cl[p]; s.f.listed = s.d.listed = on != 0; }
// the offset row ("bp", [BP_W]) or the contact-softness row ("ct", [CONTACT_W]), n leading values
int emu_cl_rows_set(void *p, const char *what, const double *v, int n) {
  Handle *h = (Handle *)p; ClSim &s = g_cl[p]; return h->fp32 ? rows_set_(h->f, s.f, what, v, n) : rows_set_(h->d, s.d, what, v, n); }
void emu_cl_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; ClSim &s = g_cl[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
// launch mode 1 (forward) or 2..6 with the rows as they are
void emu_cl_mode(void *p, int mode) { Handle *h = (Handle *)p; ClSim &s = g_cl[p]; if (h->fp32) run_(h->f, s.f, 1, mode); else run_(h->d, s.d, 1, mode); }
// the extra free body's warm start [6]
void emu_cl_set_xws(void *p, const double *v) { Handle *h = (Handle *)p; for (int i = 0; i < 6; i++) { if (h->fp32) h->f.xqacc_ws[i] = (float)v[i]; else h->d.xqacc_ws[i] = v[i]; } }
// the contact-list row [CON_W]; returns CON_W
int emu_cl_row(void *p, double *out) {
  Handle *h = (Handle *)p; ClSim &s = g_cl[p];
  for (int i = 0; i < CON_W; i++) out[i] = h->fp32 ? (double)s.f.row[i] : s.d.row[i];
  return CON_W;
}
// the frame row [count][FRAME_W]; returns count * FRAME_W
int emu_cl_frames(void *p, double *out) {
  Handle *h = (Handle *)p; ClSim &s = g_cl[p]; const int w = (h->fp32 ? s.f.nfr : s.d.nfr) * FRAME_W;
  for (int i = 0; i < w; i++) out[i] = h->fp32 ? (double)s.f.frames[i] : s.d.frames[i];
  return w;
}
}
