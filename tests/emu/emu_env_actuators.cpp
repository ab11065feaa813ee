// emu_env_actuators.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment
// actuator row (csrc/devmodel.h ACT_W) and the body-offset row the F_AC instances read with it (BP_W, holding the model's offsets).  Mode 2 runs
// step_env<..., F_ALL | F_BP | F_AC>, the source of the F_AC kernel instances (extended kind); mode 1 runs the F_BP source with the same offset row, which
// is what a batch with model-valued offset rows and no actuator rows runs; mode 0 the extended F_ALL source.  Built into its own library
// (tests/test_env_actuators.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct ActRows { real bp[BP_W], act[ACT_W]; int mode = 0; };
struct ActSim { ActRows<float> f; ActRows<double> d; };
std::map<void *, ActSim> g_ac;   // per simulator handle

template <typename real> void run_(Emu<real> &e, ActRows<real> &r, int nticks, int mode) {
  if (r.mode == 0) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.env = 0;
  if (r.mode == 1) step_env<real, true, F_ALL | F_BP>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp);
  else step_env<real, true, F_ALL | F_BP | F_AC>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act);
}
// the model's offsets in the offset row, the model's actuators (delay 6) in the actuator row: what a batch's first set gives every environment
template <typename real> void init_(Emu<real> &e, ActRows<real> &r) {
  for (int i = 0; i < BP_W; i++) r.bp[i] = i < 3 * e.hm.nbody ? (real)e.hm.body_pos[i] : real(0);
  for (int i = 0; i < ACT_W; i++) r.act[i] = 0;
  for (int i = 0; i < e.hm.nu && i < MU; i++) {
    r.act[AC_LO + i] = e.dm.act_ctrl_lo[i]; r.act[AC_HI + i] = e.dm.act_ctrl_hi[i];
    r.act[AC_WMAX + i] = (real)(e.hm.actuator_user[i] * 2 * M_PI / 60); r.act[AC_DELAY + i] = AC_MAXDELAY;
  }
}
// one environment's actuators as the batch's setter stores them: ctrlrange [nu][2], rpm [nu] (wmax formed as build_dev_model forms act_wmax), delay [nu]
// (any real: the kernel's reading of it is under test); null parts are kept
template <typename real> void set_(Emu<real> &e, ActRows<real> &r, const double *ctrlrange, const double *rpm, const double *delay) {
  for (int i = 0; i < e.hm.nu && i < MU; i++) {
    if (ctrlrange) { r.act[AC_LO + i] = (real)ctrlrange[2 * i]; r.act[AC_HI + i] = (real)ctrlrange[2 * i + 1]; }
    if (rpm) r.act[AC_WMAX + i] = (real)(rpm[i] * 2 * M_PI / 60);
    if (delay) r.act[AC_DELAY + i] = (real)delay[i];
  }
}
}  // namespace

extern "C" {
void *emu_ac_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; ActSim &s = g_ac[p]; s = ActSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_ac_free(void *p) { g_ac.erase(p); emu_free(p); }
// 0: the extended F_ALL source; 1: the F_BP source with model-valued offset rows; 2: the F_BP | F_AC source
void emu_ac_mode(void *p, int mode) { ActSim &s = g_ac[p]; s.f.mode = s.d.mode = mode; }
void emu_ac_set(void *p, const double *ctrlrange, const double *rpm, const double *delay) {
  Handle *h = (Handle *)p; ActSim &s = g_ac[p];
  if (h->fp32) set_(h->f, s.f, ctrlrange, rpm, delay); else set_(h->d, s.d, ctrlrange, rpm, delay);
}
void emu_ac_row(void *p, double *out40) {   // the actuator row as the kernel reads it
  Handle *h = (Handle *)p; ActSim &s = g_ac[p];
  for (int i = 0; i < ACT_W; i++) out40[i] = h->fp32 ? (double)s.f.act[i] : s.d.act[i];
}
void emu_ac_block(void *p, double *out30) {   // the model block's act_ctrl_lo, act_ctrl_hi, act_wmax
  Handle *h = (Handle *)p;
  for (int i = 0; i < MU; i++) {
    out30[i] = h->fp32 ? (double)h->f.dm.act_ctrl_lo[i] : h->d.dm.act_ctrl_lo[i];
    out30[10 + i] = h->fp32 ? (double)h->f.dm.act_ctrl_hi[i] : h->d.dm.act_ctrl_hi[i];
    out30[20 + i] = h->fp32 ? (double)h->f.dm.act_wmax[i] : h->d.dm.act_wmax[i];
  }
}
void emu_ac_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; ActSim &s = g_ac[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
void emu_ac_forward(void *p) { Handle *h = (Handle *)p; ActSim &s = g_ac[p]; if (h->fp32) run_(h->f, s.f, 1, 1); else run_(h->d, s.d, 1, 1); }
int emu_ac_delay_index(double v, int fp32) { return fp32 ? act_delay_index((float)v) : act_delay_index(v); }
// the batch setter's check (devbuild.h env_actuators_check): 0 accepted, 1 refused, the reason in why (at least 256 bytes)
int emu_ac_check(int n, int nu, const double *ctrlrange, const double *rpm, const int *delay, const unsigned char *mask, char *why) {
  const std::string w = env_actuators_check(n, nu, ctrlrange, rpm, delay, mask);
  snprintf(why, 256, "%s", w.c_str());
  return w.empty() ? 0 : 1;
}
}
