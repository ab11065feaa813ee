// emu_accel.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a frame table, frame rows and
// an acceleration row (csrc/devmodel.h acc_width).  With frames or the acceleration row on, a simulator runs step_env<..., F_ALL | F_FR>, the source of the
// F_FR kernel instances, on the extended instance, and then accel_row as the kernel wrapper does after a step or forward launch.  The frame table is
// built by the same host helper as cassie_batch_set_frames.  Built into its own library (tests/test_accelerations.py); never linked into, loaded by, or
// reachable from the product library.
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct AccRows { std::vector<real> tab, frames, acc; int n = 0; bool on = false; };
struct AccHandle { AccRows<float> f; AccRows<double> d; };
std::map<void *, AccHandle> g_acc;   // per simulator handle

template <typename real> void run_(Emu<real> &e, AccRows<real> &r, int nticks, int mode) {
  if (!r.n && !r.on) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.ftab = r.n ? r.tab.data() : nullptr; E.frames = r.n ? r.frames.data() : nullptr; E.nfr = r.n; E.jac = nullptr; E.jfr = 0; E.env = 0;
  step_env<real, true, F_ALL | F_FR>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
  if (r.on) accel_row(e.dm, e.sm.data(), r.acc.data(), E.ftab, E.frames, r.n, 0, e.dm.xb);   // the kernel wrapper's call after a mode-0 / mode-1 launch
}
template <typename real> int set_(Emu<real> &e, AccRows<real> &r, const char *const *names, const int *kinds, int count) {
  if (count < 0 || count > FRAME_MAX) return -1;
  std::vector<real> tab((size_t)count * FT_W);
  for (int f = 0; f < count; f++) { std::string err; if (frame_table_row(e.hm, names[f], kinds[f], &tab[(size_t)f * FT_W], err) < 0) return -1; }
  r.tab = tab; r.frames.assign((size_t)count * FRAME_W, real(0)); r.n = count;
  if (r.on) r.acc.assign(acc_width(count), real(0));   // as cassie_batch_set_frames: the new width, zero until the next launch
  return 0;
}
template <typename real> void enable_(AccRows<real> &r, int on) { r.on = on != 0; r.acc.assign(on ? acc_width(r.n) : 0, real(0)); }
template <typename real> int row_(const AccRows<real> &r, double *out) { if (!r.on) return -1; for (size_t i = 0; i < r.acc.size(); i++) out[i] = (double)r.acc[i]; return (int)r.acc.size(); }
template <typename real> int frames_(const AccRows<real> &r, double *out) { for (size_t i = 0; i < r.frames.size(); i++) out[i] = (double)r.frames[i]; return r.n; }
}  // namespace

extern "C" {
void *emu_ac_new(const char *path, int fp32) { void *p = emu_new(path, fp32); if (p) g_acc.erase(p); return p; }
void emu_ac_free(void *p) { g_acc.erase(p); emu_free(p); }
int emu_ac_set_frames(void *p, const char *const *names, const int *kinds, int count) {
  Handle *h = (Handle *)p; AccHandle &r = g_acc[p]; return h->fp32 ? set_(h->f, r.f, names, kinds, count) : set_(h->d, r.d, names, kinds, count); }
// on = 1: an acceleration row of the current frame list's width (zero until the next launch); 0: none
void emu_ac_enable(void *p, int on) { Handle *h = (Handle *)p; AccHandle &r = g_acc[p]; if (h->fp32) enable_(r.f, on); else enable_(r.d, on); }
void emu_ac_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; AccHandle &r = g_acc[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, r.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, r.d, nticks, 0); }
}
void emu_ac_forward(void *p) { Handle *h = (Handle *)p; AccHandle &r = g_acc[p]; if (h->fp32) run_(h->f, r.f, 1, 1); else run_(h->d, r.d, 1, 1); }
// the acceleration row [acc_width(count)]; returns its width, -1 without one
int emu_ac_row(void *p, double *out) { Handle *h = (Handle *)p; AccHandle &r = g_acc[p]; return h->fp32 ? row_(r.f, out) : row_(r.d, out); }
// the frame rows [count][FRAME_W]; returns count
int emu_ac_frames(void *p, double *out) { Handle *h = (Handle *)p; AccHandle &r = g_acc[p]; return h->fp32 ? frames_(r.f, out) : frames_(r.d, out); }
// the extra free body's warm start (6 entries; emu_get's qacc_ws covers the main tree)
void emu_ac_get_xws(void *p, double *out) { Handle *h = (Handle *)p; for (int i = 0; i < 6; i++) out[i] = h->fp32 ? (double)h->f.xqacc_ws[i] : h->d.xqacc_ws[i]; }
void emu_ac_set_xws(void *p, const double *in) { Handle *h = (Handle *)p; for (int i = 0; i < 6; i++) { if (h->fp32) h->f.xqacc_ws[i] = (float)in[i]; else h->d.xqacc_ws[i] = in[i]; } }
int emu_ac_width(int count) { return acc_width(count); }
}
