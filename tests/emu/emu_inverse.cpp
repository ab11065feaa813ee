// emu_inverse.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus an inverse row
// (csrc/devmodel.h INV_W).  An inverse call runs step_env in launch mode 6, then inverse_row, as the kernel wrapper does after step_env, with the caller's
// qacc in the warm-start slot: the F_ALL | F_FR source (the extended F_FR instances) on the plain handle, or the F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT
// source (f13d7 / d13d7) when the handle steps with per-environment rows (emu_env_contact.cpp's mode 2).  As cassie_batch_inverse launches it: the stage
// dump, the controller state and the counters in scratch rows, no aux row, no frames.  Built into its own library (tests/test_inverse.py); never linked into, loaded by, or reachable from
// the product library.
#include "emu_env_contact.cpp"

namespace {
struct InvRows { std::vector<float> f = std::vector<float>(INV_W); std::vector<double> d = std::vector<double>(INV_W); };
std::map<void *, InvRows> g_inv;   // per simulator handle

// qacc: [INV_COLS] by dof column (main tree 0..31, the extra free body 32..37), as the batch's "inv_qacc" row
template <typename real> void inv_(Emu<real> &e, CtRows<real> &r, const double *qacc, std::vector<real> &row) {
  // the launch's rows: the caller's qacc as the warm start, scratch stage dump, controller state and counters, no aux row, no frames
  static thread_local std::vector<real> dbg, cst; static thread_local std::vector<int> cnt;
  dbg.assign(D_SIZE, 0); cst.assign(CST_W, 0); cnt.assign(8, 0);
  EnvPtrs<real> E = e.ptrs(); E.dbg = dbg.data(); E.cst = cst.data(); E.counters = cnt.data(); E.aux = nullptr; E.ftab = nullptr; E.frames = nullptr; E.nfr = 0;
  E.jac = nullptr; E.jfr = 0; E.env = 0;
  real qa[32], xqa[32], qarow[QVEL_W_XB];   // the inverse-input row, qvel_w wide
  for (int i = 0; i < QVEL_W_XB; i++) qarow[i] = i < 32 ? (i < e.dm.nv ? (real)qacc[i] : real(0)) : (e.dm.xb >= 0 && i < 38 ? (real)qacc[i] : real(0));
  for (int i = 0; i < 32; i++) { qa[i] = qarow[i]; xqa[i] = (e.dm.xb >= 0 && i < 6) ? qarow[32 + i] : real(0); }
  if (r.mode == 0) step_env<real, true, F_ALL | F_FR>(e.dm, e.sm.data(), E, e.qvel, qa, e.xqvel, xqa, 1, 6);
  else step_env<real, true, F_ALL | F_FR | F_BP | F_AC | F_MC | F_CT>(e.dm, e.sm.data(), E, e.qvel, qa, e.xqvel, xqa, 1, 6, r.bp, r.act, r.mech, r.ct);
  inverse_row(e.dm, e.sm.data(), row.data(), E.cenv, dbg.data(), qarow, cnt.data(), 0);
}
template <typename real> void put_rows_(CtRows<real> &r, const double *bp, const double *mech) {
  if (bp) for (int i = 0; i < BP_W; i++) r.bp[i] = (real)bp[i];
  if (mech) for (int i = 0; i < MECH_W; i++) r.mech[i] = (real)mech[i];
}
}  // namespace

extern "C" {
// launch mode 6 at the current state and the given qacc [INV_COLS]: the inverse row [INV_W] into out
void emu_inv_compute(void *p, const double *qacc, double *out) {
  Handle *h = (Handle *)p; CtSim &s = g_ct[p]; InvRows &r = g_inv[p];
  if (h->fp32) { inv_(h->f, s.f, qacc, r.f); for (int i = 0; i < INV_W; i++) out[i] = r.f[i]; }
  else { inv_(h->d, s.d, qacc, r.d); for (int i = 0; i < INV_W; i++) out[i] = r.d[i]; }
}
int emu_inv_width(void) { return INV_W; }
// the body-offset row [BP_W] and the mechanics row [MECH_W] as the kernel reads them; either may be null (kept)
void emu_inv_set_rows(void *p, const double *bp, const double *mech) {
  Handle *h = (Handle *)p; CtSim &s = g_ct[p];
  if (h->fp32) put_rows_(s.f, bp, mech); else put_rows_(s.d, bp, mech);
}
void emu_inv_free(void *p) { g_inv.erase(p); emu_ct_free(p); }
}
