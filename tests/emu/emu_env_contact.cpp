// emu_env_contact.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment
// contact row (csrc/devmodel.h CONTACT_W) and the mechanics, actuator and body-offset rows the F_CT instances read with it (MECH_W, ACT_W, BP_W, holding
// the model's values).  Mode 2 runs step_env<..., F_ALL | F_BP | F_AC | F_MC | F_CT>, the source of the F_CT kernel instances (extended kind); mode 1
// runs the F_MC source with the same mechanics, actuator and offset rows, which is what a batch with model-valued mechanics rows and no contact rows
// runs; mode 0 the extended F_ALL source.
// Built into its own library (tests/test_env_contact.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct CtRows { real bp[BP_W], act[ACT_W], mech[MECH_W], ct[CONTACT_W]; int mode = 0; };
struct CtSim { CtRows<float> f; CtRows<double> d; };
std::map<void *, CtSim> g_ct;   // per simulator handle

template <typename real> void run_(Emu<real> &e, CtRows<real> &r, int nticks, int mode) {
  if (r.mode == 0) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.env = 0;
  if (r.mode == 1) step_env<real, true, F_ALL | F_BP | F_AC | F_MC>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech);
  else step_env<real, true, F_ALL | F_BP | F_AC | F_MC | F_CT>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct);
}
template <typename real> int slot_(const Emu<real> &e, int g) { return g < 256 && e.info.geom_dev[g] >= 0 && e.info.geom_dev[g] < MGT ? e.info.geom_dev[g] : -1; }
// geom g's solref, solimp and solmix into its slot (a geom without a collision slot is ignored, as the batch's setter does); null parts are kept
template <typename real> void put_(Emu<real> &e, CtRows<real> &r, int g, const double *solref, const double *solimp, const double *solmix) {
  const int s = slot_(e, g); if (s < 0) return;
  real *q = r.ct + CT_SLOT * s;
  if (solref) for (int k = 0; k < 2; k++) q[CT_SOLREF + k] = (real)solref[2 * g + k];
  if (solimp) for (int k = 0; k < 5; k++) q[CT_SOLIMP + k] = (real)solimp[5 * g + k];
  if (solmix) q[CT_SOLMIX] = (real)solmix[g];
}
// the model's offsets, actuators, mechanics and contact softness in the rows: what a batch's first set gives every environment (cassie_b200.cu)
template <typename real> void init_(Emu<real> &e, CtRows<real> &r) {
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
  for (int g = 0; g < m.ngeom; g++) put_(e, r, g, m.geom_solref.data(), m.geom_solimp.data(), m.geom_solmix.data());
}
}  // namespace

extern "C" {
void *emu_ct_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; CtSim &s = g_ct[p]; s = CtSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_ct_free(void *p) { g_ct.erase(p); emu_free(p); }
// 0: the extended F_ALL source; 1: the F_BP | F_AC | F_MC source with model-valued rows; 2: the F_BP | F_AC | F_MC | F_CT source
void emu_ct_mode(void *p, int mode) { CtSim &s = g_ct[p]; s.f.mode = s.d.mode = mode; }
int emu_ct_ngeom(void *p) { Handle *h = (Handle *)p; return h->fp32 ? h->f.hm.ngeom : h->d.hm.ngeom; }
// one environment's contact softness as the batch's setter stores it: solref [ngeom][2], solimp [ngeom][5], solmix [ngeom]; null parts are kept
void emu_ct_set(void *p, const double *solref, const double *solimp, const double *solmix) {
  Handle *h = (Handle *)p; CtSim &s = g_ct[p];
  const int ng = emu_ct_ngeom(p);
  for (int g = 0; g < ng; g++) { if (h->fp32) put_(h->f, s.f, g, solref, solimp, solmix); else put_(h->d, s.d, g, solref, solimp, solmix); }
}
void emu_ct_poke(void *p, int slot, double v) {   // one entry of the contact row, as a write through the batch's device pointer
  Handle *h = (Handle *)p; CtSim &s = g_ct[p];
  if (h->fp32) s.f.ct[slot] = (float)v; else s.d.ct[slot] = v;
}
// the model's values as the batch's get reports them without rows (the product's own compiled model), and each geom's device slot (-1: none)
void emu_ct_model(void *p, double *solref, double *solimp, double *solmix, int *slot) {
  Handle *h = (Handle *)p; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm;
  for (int g = 0; g < m.ngeom; g++) {
    for (int k = 0; k < 2; k++) solref[2 * g + k] = m.geom_solref[2 * g + k];
    for (int k = 0; k < 5; k++) solimp[5 * g + k] = m.geom_solimp[5 * g + k];
    solmix[g] = m.geom_solmix[g];
    slot[g] = h->fp32 ? slot_(h->f, g) : slot_(h->d, g);
  }
}
void emu_ct_row(void *p, double *out256) {   // the contact row as the kernel reads it
  Handle *h = (Handle *)p; CtSim &s = g_ct[p];
  for (int i = 0; i < CONTACT_W; i++) out256[i] = h->fp32 ? (double)s.f.ct[i] : s.d.ct[i];
}
void emu_ct_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; CtSim &s = g_ct[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
void emu_ct_forward(void *p) { Handle *h = (Handle *)p; CtSim &s = g_ct[p]; if (h->fp32) run_(h->f, s.f, 1, 1); else run_(h->d, s.d, 1, 1); }
// the batch setter's check (devbuild.h env_contact_check) for n environments of this model: 0 accepted, 1 refused, the reason in why (>= 512 bytes)
int emu_ct_check(void *p, int n, const double *solref, const double *solimp, const double *solmix, const unsigned char *mask, char *why) {
  Handle *h = (Handle *)p;
  const std::string w = h->fp32 ? env_contact_check(h->f.hm, n, h->f.info.geom_dev, solref, solimp, solmix, mask)
                                : env_contact_check(h->d.hm, n, h->d.info.geom_dev, solref, solimp, solmix, mask);
  snprintf(why, 512, "%s", w.c_str());
  return w.empty() ? 0 : 1;
}
}
