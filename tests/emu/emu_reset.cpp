// emu_reset.cpp -- TEST-ONLY: the product's restore source (csrc/reset.inl) compiled with -DCASSIE_EMU: the table is built by the same host helper as
// cassie_batch_reset_where / cassie_batch_set_state, and every environment runs the kernel's per-warp body with its phases as loops over 32 lanes.
// Built into its own library (tests/test_reset_where.py); never linked into, loaded by, or reachable from the product library.
#define CASSIE_EMU 1
#include "../../cassie-mujoco-sim_b200/csrc/reset.inl"

using namespace cassie;

extern "C" {
// bytes per row of each kind (RR_* order) for element size esz, qpos / qvel widths qw / vw and nframes frames; returns the number of kinds
int emu_reset_bytes(int esz, int qw, int vw, int nframes, int *bytes) { reset_row_bytes(esz, qw, vw, nframes, bytes); return RR_N; }
// one restore: dst[RR_N] the batch's rows [n][bytes] and src[RR_N] the bank's [k][bytes] (null: lacking), mask [n] (null: all), entry [n] (null: e % k).
// Returns the number of environments restored, or -1 for a table the product would refuse
int emu_reset(void *const *dst, const void *const *src, int esz, int qw, int vw, int nframes, int same_frames, const unsigned char *mask, const int *entry,
              int k, int n) {
  ResetArgs A; std::string err;
  if (!reset_table(A, dst, src, esz, qw, vw, nframes, same_frames != 0, err)) { fprintf(stderr, "emu_reset: %s\n", err.c_str()); return -1; }
  A.mask = mask; A.entry = entry; A.k = k; A.n = n;
  int count = 0;
  for (int env = 0; env < n; env++) count += reset_env(A, env) ? 1 : 0;
  return count;
}
}
