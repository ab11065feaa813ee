// emu_factor.cpp -- TEST-ONLY: the product's factor_ld (csrc/step_core.inl compiled with -DCASSIE_EMU) on matrices handed in by the test, with the
// generated Cassie-tree steps or the table-driven steps.  Built into its own library (tests/test_factor_spec.py); never linked into, loaded by, or
// reachable from the product library.
#define CASSIE_EMU 1
#include <cstdio>
#include <string>
#include <vector>
#include "../../cassie-mujoco-sim_b200/csrc/devbuild.h"
#include "../../cassie-mujoco-sim_b200/csrc/estimator_host.h"
#include "../../cassie-mujoco-sim_b200/csrc/step_core.inl"

using namespace cassie;

template <typename real> static int factor_(const char *path, int spec, const double *m, const double *m2, double *out, double *out2, double *dinv, double *dsqi, double *dinv2) {
  HostModel hm; DevModel<real> dm; std::string err;
  if (!load_model_any(path, hm, err) || !build_dev_model(hm, dm, err)) { fprintf(stderr, "emu_factor: %s\n", err.c_str()); return -1; }
  if (spec && !dm.spec19) return -2;   // the model's tree is not the one the generated code was made for
  dm.spec19 = spec;
  std::vector<real> sm(scratch_reals_ext(dm.ystride), real(0));
  real *qLD = sm.data() + S_QLD, *q2 = m2 ? sm.data() + S_Y + T_CVEL : nullptr;   // where mj_substep keeps the two matrices
  for (int a = 0; a < dm.nM; a++) { qLD[a] = (real)m[a]; if (q2) q2[a] = (real)m2[a]; }
  factor_ld<real, true>(dm, sm.data(), q2);
  for (int a = 0; a < dm.nM; a++) { out[a] = qLD[a]; if (q2) out2[a] = q2[a]; }
  for (int i = 0; i < dm.nv; i++) { dinv[i] = sm[S_DINV + i]; dsqi[i] = sm[S_DSQI + i]; if (q2) dinv2[i] = sm[S_VEC + 128 + i]; }
  return dm.nM;
}

extern "C" {
// factor M (and M2 unless null; nM entries each, in the model's sparse layout) in precision fp32 / fp64; spec: 1 the generated steps, 0 the table's.
// Out: both factors, 1/D, 1/sqrt(D) and M2's 1/D (nv each).  Returns nM, -1 when the model does not load, -2 when spec is asked of another tree
int emu_factor(const char *path, int fp32, int spec, const double *m, const double *m2, double *out, double *out2, double *dinv, double *dsqi, double *dinv2) {
  return fp32 ? factor_<float>(path, spec, m, m2, out, out2, dinv, dsqi, dinv2) : factor_<double>(path, spec, m, m2, out, out2, dinv, dsqi, dinv2);
}
}
