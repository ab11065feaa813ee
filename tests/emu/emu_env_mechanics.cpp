// emu_env_mechanics.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment
// mechanics row (csrc/devmodel.h MECH_W) and the actuator and body-offset rows the F_MC instances read with it (ACT_W, BP_W, holding the model's values).
// Mode 2 runs step_env<..., F_ALL | F_BP | F_AC | F_MC>, the source of the F_MC kernel instances (extended kind); mode 1 runs the F_AC source with the
// same actuator and offset rows, which is what a batch with model-valued actuator rows and no mechanics rows runs; mode 0 the extended F_ALL source.
// Built into its own library (tests/test_env_mechanics.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct MechRows { real bp[BP_W], act[ACT_W], mech[MECH_W]; int mode = 0; };
struct MechSim { MechRows<float> f; MechRows<double> d; };
std::map<void *, MechSim> g_mc;   // per simulator handle

template <typename real> void run_(Emu<real> &e, MechRows<real> &r, int nticks, int mode) {
  if (r.mode == 0) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.env = 0;
  if (r.mode == 1) step_env<real, true, F_ALL | F_BP | F_AC>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act);
  else step_env<real, true, F_ALL | F_BP | F_AC | F_MC>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech);
}
// the model's offsets, actuators and mechanics in the rows: what a batch's first set gives every environment (cassie_b200.cu set_env_mechanics)
template <typename real> void init_(Emu<real> &e, MechRows<real> &r) {
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
}
// one environment's mechanics as the batch's setter stores them: inertia [nbody][3], armature [nv] (main-tree dofs), stiffness / springref [njnt] (the
// hinges' go to their dof's slots); null parts are kept
template <typename real> void set_(Emu<real> &e, MechRows<real> &r, const double *inertia, const double *armature, const double *stiffness, const double *springref) {
  const HostModel &m = e.hm;
  if (inertia) for (int i = 0; i < 3 * m.nbody; i++) r.mech[MC_INERTIA + i] = (real)inertia[i];
  if (armature) for (int i = 0; i < e.dm.nv; i++) r.mech[MC_ARMATURE + i] = (real)armature[i];
  for (int j = 0; j < m.njnt; j++) {
    if (m.jnt_type[j] != JNT_HINGE) continue;
    if (stiffness) r.mech[MC_STIFF + m.jnt_dofadr[j]] = (real)stiffness[j];
    if (springref) r.mech[MC_SPRING + m.jnt_dofadr[j]] = (real)springref[j];
  }
}
template <typename real> void set_const_(Emu<real> &e, MechRows<real> &r) {   // mode 3 at qpos0 with the rows, as the batch's set_const launch
  e.enable_cenv();
  std::vector<real> keep(e.sm.begin() + S_QPOS, e.sm.begin() + S_QPOS + QPOS_W_XB);
  for (int i = 0; i < QPOS_W_XB; i++) e.sm[S_QPOS + i] = e.dm.qpos0[i];
  run_(e, r, 1, 3);
  for (int i = 0; i < QPOS_W_XB; i++) e.sm[S_QPOS + i] = keep[i];
}
}  // namespace

extern "C" {
void *emu_mc_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; MechSim &s = g_mc[p]; s = MechSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_mc_free(void *p) { g_mc.erase(p); emu_free(p); }
// 0: the extended F_ALL source; 1: the F_BP | F_AC source with model-valued rows; 2: the F_BP | F_AC | F_MC source
void emu_mc_mode(void *p, int mode) { MechSim &s = g_mc[p]; s.f.mode = s.d.mode = mode; }
void emu_mc_set(void *p, const double *inertia, const double *armature, const double *stiffness, const double *springref) {
  Handle *h = (Handle *)p; MechSim &s = g_mc[p];
  if (h->fp32) set_(h->f, s.f, inertia, armature, stiffness, springref); else set_(h->d, s.d, inertia, armature, stiffness, springref);
}
void emu_mc_poke(void *p, int slot, double v) {   // one slot of the mechanics row, as a write through the batch's device pointer
  Handle *h = (Handle *)p; MechSim &s = g_mc[p];
  if (h->fp32) s.f.mech[slot] = (float)v; else s.d.mech[slot] = v;
}
// the model's values as the batch's get reports them without rows (the product's own compiled model): inertia [nbody][3], armature [nv],
// stiffness [njnt], springref [njnt]
void emu_mc_model(void *p, double *inertia, double *armature, double *stiffness, double *springref) {
  Handle *h = (Handle *)p; const HostModel &m = h->fp32 ? h->f.hm : h->d.hm;
  for (int i = 0; i < 3 * m.nbody; i++) inertia[i] = m.body_inertia[i];
  for (int i = 0; i < m.nv; i++) armature[i] = m.dof_armature[i];
  for (int j = 0; j < m.njnt; j++) { stiffness[j] = m.jnt_stiffness[j]; springref[j] = m.qpos_spring[m.jnt_qposadr[j]]; }
}
void emu_mc_row(void *p, double *out192) {   // the mechanics row as the kernel reads it
  Handle *h = (Handle *)p; MechSim &s = g_mc[p];
  for (int i = 0; i < MECH_W; i++) out192[i] = h->fp32 ? (double)s.f.mech[i] : s.d.mech[i];
}
void emu_mc_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; MechSim &s = g_mc[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
void emu_mc_forward(void *p) { Handle *h = (Handle *)p; MechSim &s = g_mc[p]; if (h->fp32) run_(h->f, s.f, 1, 1); else run_(h->d, s.d, 1, 1); }
void emu_mc_set_const(void *p) { Handle *h = (Handle *)p; MechSim &s = g_mc[p]; if (h->fp32) set_const_(h->f, s.f); else set_const_(h->d, s.d); }
// the batch setter's check (devbuild.h env_mechanics_check) for n environments of this model: 0 accepted, 1 refused, the reason in why (>= 512 bytes)
int emu_mc_check(void *p, int n, const double *inertia, const double *armature, const double *stiffness, const double *springref, const unsigned char *mask, char *why) {
  Handle *h = (Handle *)p;
  const std::string w = h->fp32 ? env_mechanics_check(h->f.hm, n, h->f.dm.xb, h->f.dm.nv, inertia, armature, stiffness, springref, mask)
                                : env_mechanics_check(h->d.hm, n, h->d.dm.xb, h->d.dm.nv, inertia, armature, stiffness, springref, mask);
  snprintf(why, 512, "%s", w.c_str());
  return w.empty() ? 0 : 1;
}
}
