// emu_aos.cpp -- TEST-ONLY: the host emulation (emu.cpp) of the kernel instance cassie_sim_step_pd_batch runs, the plain instance plus the estimator
// stage (INST 2 in step_kernel.cuh: step_env<real, false, FEAT, true>).  emu.cpp's plain() runs the plain instance without that stage, as INST 0 does.
#include <algorithm>
#include <limits>
#include "emu.cpp"

// the plain instance's scratch on the device ends where the extended tail begins: the tail is filled with NaN, so a stage that reads it poisons the state
template <typename E> static void aos_start_(E &e) {
  e.use_ext = false; e.use_est = true; std::memset(e.est, 0, sizeof e.est);
  std::fill(e.sm.begin() + scratch_reals(e.dm.ystride), e.sm.end(), std::numeric_limits<typename decltype(e.sm)::value_type>::quiet_NaN());
}
template <typename E> static void aos_step_(E &e, const double *pd50, int nticks) {
  for (int i = 0; i < 50; i++) e.pd[i] = (typename decltype(e.sm)::value_type)pd50[i];
  step_env<typename decltype(e.sm)::value_type, false, F_ALL, true>(e.dm, e.sm.data(), e.ptrs(), e.qvel, e.qacc_ws, e.xqvel, e.xqacc_ws, nticks, 0);
}

extern "C" {
void emu_aos_start(void *p) { Handle *h = (Handle *)p; if (h->fp32) aos_start_(h->f); else aos_start_(h->d); }   // plain instance + estimator stage from now on
void emu_aos_step(void *p, const double *pd50, int nticks) { Handle *h = (Handle *)p; if (h->fp32) aos_step_(h->f, pd50, nticks); else aos_step_(h->d, pd50, nticks); }
}
