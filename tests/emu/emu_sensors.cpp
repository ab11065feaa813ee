// emu_sensors.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a per-environment sensor-model
// row (csrc/devmodel.h SN_W) and generator row (SR_W).  Mode 2 runs the chain-twin source, step_env<..., F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF |
// F_SN> with the offset, actuator, mechanics and contact rows holding the model's values and zero applied forces (what a batch with sensor rows carries
// there); mode 1 the F_XF chain twin's source with the same rows (its parent); mode 3 the plain twin's source, step_env<..., false, F_ALL | F_XF | F_SN>;
// mode 4 the plain F_XF source (its parent).  In the plain modes the scratch beyond the plain kind's size is NaN-poisoned, as emu_aos.cpp's plain mode
// does, so a read past it shows.  It also exports the generator and the draw for bitwise checks against numpy.
// Built into its own library (tests/test_sensors.py); never linked into, loaded by, or reachable from the product library.
#include <cmath>
#include <limits>
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct SnRows { real bp[BP_W], act[ACT_W], mech[MECH_W], ct[CONTACT_W], app[APPLIED_W], sn[SN_W]; int rng[SR_W]; int mode = 0; };
struct SnSim { SnRows<float> f; SnRows<double> d; };
std::map<void *, SnSim> g_sn;   // per simulator handle

template <typename real> void poison_(Emu<real> &e) {
  for (size_t i = scratch_reals(e.dm.ystride); i < e.sm.size(); i++) e.sm[i] = std::numeric_limits<real>::quiet_NaN();
}
template <typename real> void run_(Emu<real> &e, SnRows<real> &r, int nticks, int mode) {
  EnvPtrs<real> E = e.ptrs(); E.env = 0; E.ftab = nullptr; E.frames = nullptr; E.nfr = 0; E.jac = nullptr; E.jfr = 0; E.genv = nullptr;   // no frame rows
  const SensorArgs<real> sn{r.sn, r.rng};
  constexpr int CHAIN = F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT | F_XF;
  if (r.mode == 1) step_env<real, true, CHAIN>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app);
  else if (r.mode == 2) step_env<real, true, CHAIN | F_SN>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, r.bp, r.act, r.mech, r.ct, r.app, {}, {}, sn);
  else {   // the plain kind: no constant rows, no derived-quantity rows, and nothing of the extended kind's scratch
    E.aux = nullptr; E.cenv = nullptr; E.est = nullptr; E.task = nullptr; E.dbg = nullptr;
    poison_(e);
    if (r.mode == 3) step_env<real, false, F_ALL | F_XF | F_SN>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, nullptr, nullptr, nullptr, nullptr, r.app, {}, {}, sn);
    else step_env<real, false, F_ALL | F_XF>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode, nullptr, nullptr, nullptr, nullptr, r.app);
  }
}
template <typename real> int slot_(const Emu<real> &e, int g) { return g < 256 && e.info.geom_dev[g] >= 0 && e.info.geom_dev[g] < MGT ? e.info.geom_dev[g] : -1; }
// the model's offsets, actuators, mechanics and contact softness in the rows, zero applied forces, the zero sensor model, key 0 and counter 0
template <typename real> void init_(Emu<real> &e, SnRows<real> &r) {
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
  for (int i = 0; i < SN_W; i++) r.sn[i] = 0;
  r.sn[SN_QUAT] = 1;
  for (int i = 0; i < SR_W; i++) r.rng[i] = 0;
}
}  // namespace

extern "C" {
void *emu_sn_new(const char *path, int fp32) {
  void *p = emu_new(path, fp32); if (!p) return p;
  Handle *h = (Handle *)p; SnSim &s = g_sn[p]; s = SnSim();
  init_(h->f, s.f); init_(h->d, s.d);
  return p;
}
void emu_sn_free(void *p) { g_sn.erase(p); emu_free(p); }
// 1: the F_XF chain twin's source (parent); 2: the chain twin; 3: the plain twin; 4: the plain F_XF source (parent)
void emu_sn_mode(void *p, int mode) { SnSim &s = g_sn[p]; s.f.mode = s.d.mode = mode; }
// one environment's sensor row as the kernel reads it ([SN_W], devmodel.h layout, the quaternion as given) and its generator (key, counter)
void emu_sn_set_row(void *p, const double *row, unsigned long long key, unsigned long long counter) {
  Handle *h = (Handle *)p; SnSim &s = g_sn[p];
  for (int i = 0; i < SN_W; i++) { s.f.sn[i] = (float)row[i]; s.d.sn[i] = row[i]; }
  const int g[SR_W] = {(int)(uint32_t)key, (int)(uint32_t)(key >> 32), (int)(uint32_t)counter, (int)(uint32_t)(counter >> 32)};
  for (int i = 0; i < SR_W; i++) { s.f.rng[i] = g[i]; s.d.rng[i] = g[i]; }
  (void)h;
}
unsigned long long emu_sn_counter(void *p) { Handle *h = (Handle *)p; const int *g = h->fp32 ? g_sn[p].f.rng : g_sn[p].d.rng; return (unsigned long long)(uint32_t)g[2] | ((unsigned long long)(uint32_t)g[3] << 32); }
void emu_sn_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; SnSim &s = g_sn[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, s.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, s.d, nticks, 0); }
}
void emu_sn_forward(void *p) { Handle *h = (Handle *)p; SnSim &s = g_sn[p]; if (h->fp32) run_(h->f, s.f, 1, 1); else run_(h->d, s.d, 1, 1); }
// the generator: blocks (t[i], j[i]) of key[i], 4 words each
void emu_sn_philox(const unsigned long long *t, const unsigned long long *j, const unsigned long long *key, unsigned long long *out, int count) {
  for (int i = 0; i < count; i++) { uint64_t w[4]; philox4x64_10(t[i], j[i], key[i], w[0], w[1], w[2], w[3]); for (int k = 0; k < 4; k++) out[4 * i + k] = w[k]; }
}
// the draws of std sigma[i] from word[i], in fp32 (out32) and fp64 (out64)
void emu_sn_noise(const double *sigma, const unsigned long long *word, float *out32, double *out64, int count) {
  for (int i = 0; i < count; i++) { out32[i] = sn_noise<float>((float)sigma[i], word[i]); out64[i] = sn_noise<double>(sigma[i], word[i]); }
}
}
