// env_rows.h -- which per-environment row blocks a batch holds because another block needs them, and when they go.  Host code without CUDA:
// cassie_b200.cu runs every setter, clear and launch of the blocks through it, tests/test_env_rows.py compiles it with g++.
//
// The step-kernel instances of the blocks are nested twins (step_instances.inc): an instance that reads one block also reads the block it needs, so
// a batch that holds a block also holds what it needs.  Where the caller has not set a needed block, it is lent: allocated holding the model's
// values (applied forces: zero) and marked lent.  A setter makes a block the caller's; dropping a block releases what it had lent, down the chain.
#pragma once

namespace cassie {

enum RowBlock { R_CENV, R_BPOS, R_ACT, R_MECH, R_CT, R_APP, R_TRACE, R_CL, R_SN, R_N };   // in chain order
enum RowWhen { AT_SET = 1, AT_LAUNCH = 2, AT_EXT_LAUNCH = 4 };   // when the need is lent: at the block's set, at every launch, at extended launches

// need: the block it needs; when: RowWhen bits; keep: its own clear keeps it (model values, lent) while a block that needs it is present, instead
// of dropping it; ext: its launches are extended, so what its need needs at extended launches is lent with it
struct RowLink { int need, when; bool keep, ext; };
constexpr RowLink ROW_LINKS[R_N] = {
  {-1, 0, false, false},                    // constant rows (A.cenv): set_model_rows, get_model_rows and set_const allocate them too
  {R_CENV, AT_SET, true, false},            // body offsets: set_const writes their invweights into the constant rows
  {R_BPOS, AT_SET, true, false},            // actuators
  {R_ACT, AT_SET, true, false},             // mechanics
  {R_MECH, AT_SET, false, false},           // contact softness
  {R_CT, AT_EXT_LAUNCH, false, false},      // applied forces: the plain twins f0404 / f2404 read no contact rows, the extended chain twins do
  {R_APP, AT_SET | AT_LAUNCH, false, true},   // per-tick trace
  {R_APP, AT_SET | AT_LAUNCH, false, true},   // contact lists
  {R_APP, AT_SET | AT_LAUNCH, false, false},  // sensor models
};

enum RowOp { ROW_LEND, ROW_MODEL, ROW_DROP };   // allocate holding the model's values, lent / rewrite to the model's values, lent / free
struct RowStep { int op, block; };
struct RowPlan { int n = 0; RowStep step[4 * R_N]; void add(int op, int b) { step[n++] = {op, b}; } };   // what the batch does, in order
struct RowState {
  unsigned have = 0, lent = 0;   // bit per RowBlock: the rows exist / they were lent, and no setter has written them since
  bool has(int b) const { return (have >> b) & 1; }
  bool is_lent(int b) const { return (lent >> b) & 1; }
};

// b present, and what it needs at set (with ext: at extended launches too); absent blocks are lent, needs first
inline void provide(RowState &s, RowPlan &p, int b, bool ext) {
  const RowLink &l = ROW_LINKS[b];
  if (!s.has(b)) {
    if (l.need >= 0 && (l.when & AT_SET)) provide(s, p, l.need, ext);
    s.have |= 1u << b; s.lent |= 1u << b; p.add(ROW_LEND, b);
  }
  if (l.need >= 0 && ext && (l.when & AT_EXT_LAUNCH)) provide(s, p, l.need, ext);
}

// a setter of b: what b needs is lent where absent, and b is the caller's (the setter allocates it when absent)
inline void own(RowState &s, RowPlan &p, int b) {
  const RowLink &l = ROW_LINKS[b];
  if (l.need >= 0 && (l.when & AT_SET)) provide(s, p, l.need, l.ext);
  s.have |= 1u << b; s.lent &= ~(1u << b);
}

inline void dropped(RowState &s, RowPlan &p, int b);

// b's clear: kept holding the model's values while a block that needs it is present and its link says keep, else dropped
inline void release(RowState &s, RowPlan &p, int b) {
  if (!s.has(b)) return;
  bool held = false;
  for (int d = 0; d < R_N; d++) held |= s.has(d) && ROW_LINKS[d].need == b;
  if (ROW_LINKS[b].keep && held) { s.lent |= 1u << b; p.add(ROW_MODEL, b); return; }
  p.add(ROW_DROP, b);
  dropped(s, p, b);
}

// b is gone (dropped here, or freed by its own verb): what it had lent is released
inline void dropped(RowState &s, RowPlan &p, int b) {
  s.have &= ~(1u << b); s.lent &= ~(1u << b);
  const int need = ROW_LINKS[b].need;
  if (need >= 0 && s.is_lent(need)) release(s, p, need);
}

// before a launch of `kind` (1: extended): what the present blocks need at launch, lent where a verb dropped it since their set
inline void lend_for_launch(RowState &s, RowPlan &p, int kind) {
  const bool ext = kind == 1;
  for (int b = R_N - 1; b >= 0; b--) {
    const RowLink &l = ROW_LINKS[b];
    if (s.has(b) && l.need >= 0 && ((l.when & AT_LAUNCH) || (ext && (l.when & AT_EXT_LAUNCH)))) provide(s, p, l.need, ext || l.ext);
  }
}

// an extended launch would lend rows for a block's extended-launch link (forward_where allocates nothing, so it refuses that launch)
inline bool launch_lends_ext(const RowState &s, bool ext) {
  for (int b = 0; ext && b < R_N; b++)
    if (s.has(b) && (ROW_LINKS[b].when & AT_EXT_LAUNCH) && !s.has(ROW_LINKS[b].need)) return true;
  return false;
}

// cassie_sim_copy: the model blocks the source lacks are cleared top down, then the source's model blocks come with their lent bits.  Applied
// forces are state, not model: they are not copied
constexpr unsigned ROW_MODEL_BLOCKS = (1u << R_APP) - 1;
inline void copy_from(RowState &s, RowPlan &p, const RowState &src) {
  for (int b = R_APP - 1; b > R_CENV; b--) if (!src.has(b)) release(s, p, b);
  const unsigned m = src.have & ROW_MODEL_BLOCKS;
  s.have = (s.have & ~ROW_MODEL_BLOCKS) | m; s.lent = (s.lent & ~m) | (src.lent & m);
}

}  // namespace cassie
