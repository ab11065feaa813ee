// emu_trace.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) with the per-tick trace of the
// F_TC instances.  A simulator runs the trace twin's source, step_env<..., F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF | F_TC>, with the offset,
// actuator, mechanics and contact rows holding the model's values and zero applied forces (what a traced batch carries there), an optional frame
// table and a trace row [T][k]; or, untraced, the chain twin's source (the same without F_TC) on the same rows.  The aux row stays as emu.cpp has it
// (on).  Built into its own library (tests/test_trace.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <map>
#include "emu.cpp"

namespace {
constexpr int CHAIN = F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF;
template <typename real> struct TcRows {
  real bp[BP_W], act[ACT_W], mech[MECH_W], ct[CONTACT_W], app[APPLIED_W];
  std::vector<real> ftab, frames, trace; std::vector<int> cols; int nfr = 0, k = 0, T = 0, need = 0; bool traced = true;
};
struct TcSim { TcRows<float> f; TcRows<double> d; };
std::map<void *, TcSim> g_tc;   // per simulator handle

template <typename real> void run_(Emu<real> &e, TcRows<real> &r, int nticks, int mode) {
  EnvPtrs<real> E = e.ptrs(); E.env = 0; E.genv = nullptr; E.jac = nullptr; E.jfr = 0;
  E.ftab = r.nfr ? r.ftab.data() : nullptr; E.frames = r.nfr ? r.frames.data() : nullptr; E.nfr = r.nfr;
  if (r.traced && r.k > 0) {
    const TraceArgs<real> tr{r.trace.data(), r.cols.data(), r.k, r.T, r.need};
    step_env<real, true, CHAIN | F_TC>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app, tr);
  } else {
    step_env<real, true, CHAIN>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app);
  }
}
template <typename real> int slot_(const Emu<real> &e, int g) { return g < 256 && e.info.geom_dev[g] >= 0 && e.info.geom_dev[g] < MGT ? e.info.geom_dev[g] : -1; }
// the model's offsets, actuators, mechanics and contact softness in the rows, zero applied forces (as emu_applied_forces.cpp)
template <typename real> void init_(Emu<real> &e, TcRows<real> &r) {
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
template <typename real> int frames_(Emu<real> &e, TcRows<real> &r, const char *const *names, const int *kinds, int count) {
  if (count < 0 || count > FRAME_MAX) return -1;
  std::vector<real> tab((size_t)count * FT_W);
  for (int f = 0; f < count; f++) { std::string err; if (frame_table_row(e.hm, names[f], kinds[f], &tab[(size_t)f * FT_W], err) < 0) return -1; }
  r.ftab = tab; r.frames.assign((size_t)count * FRAME_W, real(0)); r.nfr = count;
  return 0;
}
// the column table as cassie_batch_set_trace builds it (the host checks are the product's; here the sources are trusted)
template <typename real> void trace_(TcRows<real> &r, const int *src, const int *col, int k, int T) {
  r.k = k; r.T = T; r.need = 0; r.cols.assign((size_t)k, 0); r.trace.assign((size_t)k * T, real(0));
  for (int c = 0; c < k; c++) { r.cols[c] = (src[c] << TC_SHIFT) | col[c]; if (src[c] >= TC_OBS) r.need |= 1 << src[c]; }
}
}  // namespace

extern "C" {
void *emu_tc_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; TcSim &s = g_tc[p]; s = TcSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_tc_free(void *p) { g_tc.erase(p); emu_free(p); }
int emu_tc_set_frames(void *p, const char *const *names, const int *kinds, int count) {
  Handle *h = (Handle *)p; TcSim &s = g_tc[p]; return h->fp32 ? frames_(h->f, s.f, names, kinds, count) : frames_(h->d, s.d, names, kinds, count); }
// k columns (source, column) and T slots; k = 0: no trace.  traced = 0 runs the chain twin's source instead (the same rows, no F_TC)
void emu_tc_set_trace(void *p, const int *src, const int *col, int k, int T) { TcSim &s = g_tc[p]; trace_(s.f, src, col, k, T); trace_(s.d, src, col, k, T); }
void emu_tc_traced(void *p, int on) { TcSim &s = g_tc[p]; s.f.traced = s.d.traced = on != 0; }
void emu_tc_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; TcSim &s = g_tc[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
void emu_tc_forward(void *p) { Handle *h = (Handle *)p; TcSim &s = g_tc[p]; if (h->fp32) run_(h->f, s.f, 1, 1); else run_(h->d, s.d, 1, 1); }
// the trace row [T][k]; returns T * k
int emu_tc_trace(void *p, double *out) {
  Handle *h = (Handle *)p; TcSim &s = g_tc[p]; const int w = h->fp32 ? s.f.k * s.f.T : s.d.k * s.d.T;
  for (int i = 0; i < w; i++) out[i] = h->fp32 ? (double)s.f.trace[i] : s.d.trace[i];
  return w;
}
// the frame row [count][FRAME_W]; returns count * FRAME_W
int emu_tc_frames(void *p, double *out) {
  Handle *h = (Handle *)p; TcSim &s = g_tc[p]; const int w = (h->fp32 ? s.f.nfr : s.d.nfr) * FRAME_W;
  for (int i = 0; i < w; i++) out[i] = h->fp32 ? (double)s.f.frames[i] : s.d.frames[i];
  return w;
}
}
