// step_select.h -- which compiled instance of the fused step kernel a launch runs.  Host code without CUDA: cassie_b200.cu picks its launches
// with it, tests/test_step_instances.py compiles it with g++.  The instances are the lines of step_instances.inc.
#pragma once
#include "devmodel.h"

namespace cassie {

struct StepInstance { bool dbl; int kind, feat; const void *(*entry)(void); };   // kind: 0 plain, 1 extended, 2 plain + estimator

// the instance a tag of step_instances.inc names: <f|d><kind digit><feature bits in hex>; entry is its cassie_step_entry_<tag> (step_inst.cu)
constexpr StepInstance step_instance(const char *tag, const void *(*entry)(void) = nullptr) {
  int feat = 0;
  for (const char *c = tag + 2; *c; ++c) feat = 16 * feat + (*c <= '9' ? *c - '0' : *c - 'a' + 10);
  return {tag[0] == 'd', tag[1] - '0', feat, entry};
}

struct StepChoice { int kind, index; };   // the kind a launch runs and its instance in the table (-1: none compiled)

// the instance for a launch of `kind` asking for the features `feat`: among the table's instances of that precision and kind, the one with every
// requested feature and the fewest bits set.  Applied forces (F_XF) stay on a plain kind only for a box-only model with a plain twin (f0404 /
// f2404 and their F_SN twins, the push workload); every other request with them runs the extended kind.
inline StepChoice step_select(const StepInstance *table, int n, bool dbl, int kind, int feat) {
  auto cover = [&](int k) {
    int best = -1;
    for (int i = 0; i < n; i++)
      if (table[i].dbl == dbl && table[i].kind == k && (table[i].feat & feat) == feat && (best < 0 || __builtin_popcount(table[i].feat) < __builtin_popcount(table[best].feat))) best = i;
    return best;
  };
  if (kind != 1 && (feat & F_XF)) {
    const int i = (feat & F_ALL) == F_BOX ? cover(kind) : -1;
    if (i >= 0) return {kind, i};
    kind = 1;
  }
  return {kind, cover(kind)};
}

}  // namespace cassie
