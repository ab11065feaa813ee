// emu_dynamics.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a dynamics row
// (csrc/devmodel.h DYN_W).  A dynamics call runs step_env<..., F_ALL | F_FR> in launch mode 5, the source of the F_FR kernel instances, on the extended
// instance without frames and without the debug row, as cassie_batch_dynamics launches it.  Stepping stays on emu.cpp's instance.  Built into its own
// library (tests/test_dynamics.py); never linked into, loaded by, or reachable from the product library.
#include <map>
#include "emu.cpp"

namespace {
struct DynRows { std::vector<float> f = std::vector<float>(DYN_W); std::vector<double> d = std::vector<double>(DYN_W); };
std::map<void *, DynRows> g_dyn;   // per simulator handle

template <typename real> void dyn_(Emu<real> &e, std::vector<real> &row) {
  EnvPtrs<real> E = e.ptrs(); E.dbg = nullptr; E.ftab = nullptr; E.frames = nullptr; E.nfr = 0; E.jac = nullptr; E.jfr = 0; E.env = 0;
  step_env<real, true, F_ALL | F_FR>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, 1, 5);
  dynamics_row(e.dm, e.sm.data(), row.data(), E.cenv, 0, e.dm.xb);   // as the kernel wrapper does after step_env
}
}  // namespace

extern "C" {
void *emu_dyn_new(const char *path, int fp32) { void *p = emu_new(path, fp32); if (p) g_dyn.erase(p); return p; }
void emu_dyn_free(void *p) { g_dyn.erase(p); emu_free(p); }
// launch mode 5 at the current state: the dynamics row [DYN_W] into out
void emu_dyn_compute(void *p, double *out) {
  Handle *h = (Handle *)p; DynRows &r = g_dyn[p];
  if (h->fp32) { dyn_(h->f, r.f); for (int i = 0; i < DYN_W; i++) out[i] = r.f[i]; }
  else { dyn_(h->d, r.d); for (int i = 0; i < DYN_W; i++) out[i] = r.d[i]; }
}
int emu_dyn_width(void) { return DYN_W; }
}
