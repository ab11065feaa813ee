// emu_applied_forces.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment
// applied-force row (csrc/devmodel.h APPLIED_W: xfrc_applied [32][6], qfrc_applied [40]).  Mode 2 runs the chain-twin source, step_env<..., F_ALL | F_BP |
// F_AC | F_MC | F_CT | F_XF> with the offset, actuator, mechanics and contact rows holding the model's values (what a batch with applied rows carries
// there); mode 1 the F_CT source with the same rows (the chain twin's parent); mode 3 the plain twin's source, step_env<..., false, F_ALL | F_XF> (the
// plain kind: no per-environment constants, no derived-quantity rows); mode 4 the plain F_ALL source (its parent); mode 0 the extended F_ALL source.
// In the plain modes the scratch beyond the plain kind's size is NaN-poisoned, as emu_aos.cpp's plain mode does, so a read past it shows.
// Built into its own library (tests/test_applied_forces.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <limits>
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct XfRows { real bp[BP_W], act[ACT_W], mech[MECH_W], ct[CONTACT_W], app[APPLIED_W]; int mode = 0; };
struct XfSim { XfRows<float> f; XfRows<double> d; };
std::map<void *, XfSim> g_xf;   // per simulator handle

template <typename real> void poison_(Emu<real> &e) {
  for (size_t i = scratch_reals(e.dm.ystride); i < e.sm.size(); i++) e.sm[i] = std::numeric_limits<real>::quiet_NaN();
}
template <typename real> void run_(Emu<real> &e, XfRows<real> &r, int nticks, int mode) {
  if (r.mode == 0) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.env = 0; E.ftab = nullptr; E.frames = nullptr; E.nfr = 0; E.jac = nullptr; E.jfr = 0; E.genv = nullptr;   // no frame rows
  if (r.mode == 1) step_env<real, true, F_ALL | F_BP | F_AC | F_MC | F_CT>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct);
  else if (r.mode == 2) step_env<real, true, F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app);
  else {   // the plain kind: no constant rows, no derived-quantity rows, and nothing of the extended kind's scratch
    E.aux = nullptr; E.cenv = nullptr; E.est = nullptr; E.task = nullptr; E.dbg = nullptr;
    poison_(e);
    if (r.mode == 3) step_env<real, false, F_ALL | F_XF>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, nullptr, nullptr, nullptr, nullptr, r.app);
    else step_env<real, false, F_ALL>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
  }
}
template <typename real> int slot_(const Emu<real> &e, int g) { return g < 256 && e.info.geom_dev[g] >= 0 && e.info.geom_dev[g] < MGT ? e.info.geom_dev[g] : -1; }
// the model's offsets, actuators, mechanics and contact softness in the rows (what the batch's carried rows hold), zero applied forces
template <typename real> void init_(Emu<real> &e, XfRows<real> &r) {
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
  for (int g = 0; g < m.ngeom; g++) {
    const int s = slot_(e, g); if (s < 0) continue;
    real *q = r.ct + CT_SLOT * s;
    for (int k = 0; k < 2; k++) q[CT_SOLREF + k] = (real)m.geom_solref[2 * g + k];
    for (int k = 0; k < 5; k++) q[CT_SOLIMP + k] = (real)m.geom_solimp[5 * g + k];
    q[CT_SOLMIX] = (real)m.geom_solmix[g];
  }
  for (int i = 0; i < APPLIED_W; i++) r.app[i] = 0;
}
}  // namespace

extern "C" {
void *emu_xf_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; XfSim &s = g_xf[p]; s = XfSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_xf_free(void *p) { g_xf.erase(p); emu_free(p); }
// 0: the extended F_ALL source; 1: the F_CT source (chain parent); 2: the chain twin; 3: the plain twin; 4: the plain F_ALL source (plain parent)
void emu_xf_mode(void *p, int mode) { XfSim &s = g_xf[p]; s.f.mode = s.d.mode = mode; }
// one environment's applied-force row as the kernel reads it ([APPLIED_W]: xfrc_applied [32][6] in model body order, qfrc_applied [40] by column)
void emu_xf_set_row(void *p, const double *row) {
  Handle *h = (Handle *)p; XfSim &s = g_xf[p];
  for (int i = 0; i < APPLIED_W; i++) { if (h->fp32) s.f.app[i] = (float)row[i]; else s.d.app[i] = row[i]; }
}
void emu_xf_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; XfSim &s = g_xf[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
// mode 5 (the dynamics launch) at the current state: the bias forces qfrc_bias [nv main-tree dofs] it leaves for the dynamics row (fp64 handles only)
int emu_xf_bias(void *p, double *out) {
  Handle *h = (Handle *)p; XfSim &s = g_xf[p];
  if (h->fp32 || s.d.mode != 2) return -1;
  run_(h->d, s.d, 1, 5);
  for (int i = 0; i < h->d.dm.nv; i++) out[i] = h->d.sm[S_VEC + 32 + i];
  return h->d.dm.nv;
}
}
