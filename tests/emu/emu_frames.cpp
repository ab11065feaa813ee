// emu_frames.cpp -- TEST-ONLY: the host emulation of emu.cpp (the product's step_core.inl compiled with -DCASSIE_EMU) plus a frame table and a frame
// row (csrc/devmodel.h FRAME_W).  With frames set, a simulator runs step_env<..., F_ALL | F_FR>, the source of the F_FR kernel instances, on the
// extended instance (the aux row stays as emu.cpp has it: on, or off after emu_plain).  The table is built by the same host helper as
// cassie_batch_set_frames.  Built into its own library (tests/test_frames.py); never linked into, loaded by, or reachable from the product library.
#include <map>
#include "emu.cpp"

namespace {
template <typename real> struct FrameRow { std::vector<real> tab, row, jac = std::vector<real>(FRAME_JAC_W); int n = 0, jfr = 0; };
struct FrameRows { FrameRow<float> f; FrameRow<double> d; };
std::map<void *, FrameRows> g_frames;   // per simulator handle

template <typename real> void run_(Emu<real> &e, FrameRow<real> &r, int nticks, int mode) {
  if (!r.n) { e.run(nticks, mode); return; }
  EnvPtrs<real> E = e.ptrs(); E.ftab = r.tab.data(); E.frames = r.row.data(); E.nfr = r.n; E.jac = r.jac.data(); E.jfr = r.jfr; E.env = 0;
  step_env<real, true, F_ALL | F_FR>(e.dm, e.sm.data(), E, e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, mode);
}
template <typename real> int set_(Emu<real> &e, FrameRow<real> &r, const char *const *names, const int *kinds, int count) {
  if (count < 0 || count > FRAME_MAX) return -1;
  std::vector<real> tab((size_t)count * FT_W);
  for (int f = 0; f < count; f++) { std::string err; if (frame_table_row(e.hm, names[f], kinds[f], &tab[(size_t)f * FT_W], err) < 0) return -1; }
  r.tab = tab; r.row.assign((size_t)count * FRAME_W, real(0)); r.n = count;
  return 0;
}
}  // namespace

extern "C" {
void *emu_fr_new(const char *path, int fp32) { void *p = emu_new(path, fp32); if (p) g_frames.erase(p); return p; }
void emu_fr_free(void *p) { g_frames.erase(p); emu_free(p); }
int emu_fr_set(void *p, const char *const *names, const int *kinds, int count) {
  Handle *h = (Handle *)p; FrameRows &r = g_frames[p]; return h->fp32 ? set_(h->f, r.f, names, kinds, count) : set_(h->d, r.d, names, kinds, count); }
void emu_fr_step(void *p, const double *pd50, int nticks) {
  Handle *h = (Handle *)p; FrameRows &r = g_frames[p];
  if (h->fp32) { for (int i = 0; i < 50; i++) h->f.pd[i] = (float)pd50[i]; run_(h->f, r.f, nticks, 0); }
  else { for (int i = 0; i < 50; i++) h->d.pd[i] = pd50[i]; run_(h->d, r.d, nticks, 0); }
}
void emu_fr_forward(void *p) { Handle *h = (Handle *)p; FrameRows &r = g_frames[p]; if (h->fp32) run_(h->f, r.f, 1, 1); else run_(h->d, r.d, 1, 1); }
// launch mode 4 for frame f: the Jacobian row [6][FJ_COLS] at the current state into out; -1 for a frame out of range
int emu_fr_jacobian(void *p, int f, double *out) {
  Handle *h = (Handle *)p; FrameRows &r = g_frames[p]; const int n = h->fp32 ? r.f.n : r.d.n;
  if (f < 0 || f >= n) return -1;
  if (h->fp32) { r.f.jfr = f; run_(h->f, r.f, 1, 4); } else { r.d.jfr = f; run_(h->d, r.d, 1, 4); }
  for (int i = 0; i < FRAME_JAC_W; i++) out[i] = h->fp32 ? (double)r.f.jac[i] : r.d.jac[i];
  return 0;
}
// the frame row [count][FRAME_W]; returns count
int emu_fr_row(void *p, double *out) {
  Handle *h = (Handle *)p; FrameRows &r = g_frames[p]; const int n = h->fp32 ? r.f.n : r.d.n;
  for (int i = 0; i < n * FRAME_W; i++) out[i] = h->fp32 ? (double)r.f.row[i] : r.d.row[i];
  return n;
}
}
