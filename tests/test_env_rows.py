"""The lending rule of the per-environment row blocks (csrc/env_rows.h), compiled on the host with g++ (no GPU, no CUDA headers).

tests/golden/env_rows_transcript.json.gz holds what a batch did after every verb of many sequences (tests/golden/make_env_rows_transcript.py).  A
harness replays the accepted verbs through the header and must predict every recorded row pointer and every refusal that depends on the batch's
rows.  Independently of the transcript, every verb sequence up to length 4 must leave each present block with the blocks it needs, and a set
followed by its clear must restore the state before the set wherever the table says it does."""
import gzip
import itertools
import json
import os
import subprocess

import pytest

from conftest import GOLDEN, REPO

CSRC = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'csrc')
MODEL_FEAT = {'cassie': 4, 'cassie_tray_box': 5}   # F_BOX / F_XB | F_BOX: the features Batch::init derives from the models


# stdin: one case per line, "<feat> <dbl> <legacy> <copy> verb...": copy 1 replays the verbs on a cassie_sim_t's batch, then copies it into a fresh
# one (verb "copy") whose forward follows.  stdout per verb: accepted (0/1), the pointer bits of actuators, mechanics, contact, applied, trace,
# contacts, sensors, and the state's have and lent words
HARNESS = r'''
#include <cstdio>
#include <cstring>
#include <iostream>
#include <sstream>
#include <string>
#include "step_select.h"
#include "env_rows.h"
using namespace cassie;
static const StepInstance TABLE[] = {
#define STEP_INSTANCE(tag) step_instance(#tag),
#include "step_instances.inc"
#undef STEP_INSTANCE
};
static const int NT = sizeof TABLE / sizeof TABLE[0];
struct Sim { RowState s; int feat = 0; bool dbl = false, aux = false, snap = false, snap_app = false; };
static int feat_of(const Sim &b) {   // Batch::launch_feat
  static const int bit[R_N] = {0, F_BP, F_AC, F_MC, F_CT, F_XF, F_TC, F_CL, F_SN};
  int f = b.feat | (b.s.has(R_CL) ? F_FR : 0);
  for (int r = 0; r < R_N; r++) if (b.s.has(r)) f |= bit[r];
  return f;
}
static int kind_of(const Sim &b, int mode) {   // Batch::launch_kind for the rows the transcript's verbs make
  const RowState &s = b.s;
  const int ext = (s.has(R_CENV) || b.aux || s.has(R_TRACE) || s.has(R_CL) || mode >= 3) ? 1 : 0;
  return step_select(TABLE, NT, b.dbl, ext, feat_of(b)).kind;
}
static bool launch(Sim &b, int mode) {   // false: no instance covers the rows once lent (step_range's refusal)
  const int kind = kind_of(b, mode); RowPlan p; lend_for_launch(b.s, p, kind);
  const StepChoice c = step_select(TABLE, NT, b.dbl, kind, feat_of(b));
  return c.kind == kind && c.index >= 0;
}
static bool play(Sim &b, const std::string &v) {   // false: refused
  RowState &s = b.s; RowPlan p;
  const char *own_v[] = {"set_bpos", "set_act", "set_mech", "set_ct", "set_ct_null", "set_app", "app_on"};
  const int own_b[] = {R_BPOS, R_ACT, R_MECH, R_CT, R_CT, R_APP, R_APP};
  for (int i = 0; i < 7; i++) if (v == own_v[i]) { own(s, p, own_b[i]); return true; }
  const char *clr_v[] = {"clear_bpos", "clear_act", "clear_mech", "clear_ct"};
  for (int i = 0; i < 4; i++) if (v == clr_v[i]) { release(s, p, R_BPOS + i); return true; }
  if (v == "app_off") { dropped(s, p, R_APP); return true; }
  if (v == "set_sn") { if (s.has(R_TRACE) || s.has(R_CL)) return false; if (!s.has(R_SN)) own(s, p, R_SN); return true; }
  if (v == "clear_sn") { if (s.has(R_SN)) dropped(s, p, R_SN); return true; }
  if (v == "set_model_rows") { own(s, p, R_CENV); return true; }
  if (v == "get_model_rows") { s.have |= 1u << R_CENV; return true; }
  if (v == "trace_on") { if (s.has(R_CL) || s.has(R_SN)) return false; own(s, p, R_TRACE); return true; }
  if (v == "trace_off") { dropped(s, p, R_TRACE); return true; }
  if (v == "cl_on") { if (s.has(R_TRACE) || s.has(R_SN)) return false; if (!s.has(R_CL)) own(s, p, R_CL); return true; }
  if (v == "cl_off") { if (s.has(R_CL)) dropped(s, p, R_CL); return true; }
  if (v == "aux_on" || v == "aux_off") { b.aux = v == "aux_on"; return true; }
  if (v == "step") { launch(b, 0); return true; }   // (cassie_batch_step and cassie_batch_forward report nothing)
  if (v == "forward") { launch(b, 1); return true; }
  if (v == "set_const") { s.have |= 1u << R_CENV; return launch(b, 3); }
  if (v == "forward_where") { if (launch_lends_ext(s, kind_of(b, 1) == 1)) return false; return launch(b, 1); }
  if (v == "get_state") { b.snap = true; b.snap_app = s.has(R_APP); return true; }
  if (v == "set_state") { if (!b.snap) { b.snap = true; b.snap_app = s.has(R_APP); } if (b.snap_app && !s.has(R_APP)) own(s, p, R_APP); return true; }
  if (v == "bad_set") return false;
  fprintf(stderr, "unknown verb %s\n", v.c_str()); return false;
}
static void out(const Sim &b, bool ok) {
  const int r[7] = {R_ACT, R_MECH, R_CT, R_APP, R_TRACE, R_CL, R_SN};
  printf("%d ", ok); for (int i = 0; i < 7; i++) printf("%d", b.s.has(r[i])); printf(" %u %u\n", b.s.have, b.s.lent);
}
int main() {
  std::string line;
  while (std::getline(std::cin, line)) {
    std::istringstream in(line); int feat, dbl, legacy, copy; in >> feat >> dbl >> legacy >> copy;
    Sim b; b.feat = feat; b.dbl = dbl; b.aux = legacy;   // a cassie_sim_t's batch carries derived-quantity rows
    std::string v;
    while (in >> v) out(b, play(b, v));
    if (copy) {   // cassie_sim_copy into a fresh simulator, then its forward
      Sim d; d.feat = feat; d.dbl = dbl; d.aux = true; RowPlan p;
      copy_from(d.s, p, b.s);
      if (b.s.has(R_SN) && !d.s.has(R_SN)) own(d.s, p, R_SN);
      if (b.s.has(R_APP) && !d.s.has(R_APP)) own(d.s, p, R_APP);   // the state copy (cassie_set_state) restores a snapshot with applied rows
      out(d, true);
      out(d, play(d, "forward"));
    }
    printf("end\n"); fflush(stdout);
  }
}
'''


@pytest.fixture(scope='module')
def harness(tmp_path_factory):
    tmp = tmp_path_factory.mktemp('env_rows')
    src, exe = tmp / 'rows.cpp', tmp / 'rows'
    src.write_text(HARNESS)
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-I', CSRC, '-o', str(exe), str(src)])

    def run(cases):
        """cases: [(feat, dbl, legacy, copy, verbs)] -> per case [(ok, pointer bits, have, lent)] per verb"""
        text = ''.join('%d %d %d %d %s\n' % (f, d, lg, c, ' '.join(v)) for f, d, lg, c, v in cases)
        lines = subprocess.run([str(exe)], input=text, capture_output=True, text=True, check=True).stdout.splitlines()
        res, cur = [], []
        for ln in lines:
            if ln == 'end':
                res.append(cur)
                cur = []
            else:
                ok, bits, have, lent = ln.split()
                cur.append((ok == '1', bits, int(have), int(lent)))
        return res
    return run


@pytest.fixture(scope='module')
def transcript():
    with gzip.open(os.path.join(GOLDEN, 'env_rows_transcript.json.gz'), 'rt') as f:
        return json.load(f)


def test_transcript_is_replayed_by_the_rule(harness, transcript):
    """every recorded pointer bit and every refusal that depends on the batch's rows, forward_where's included; value refusals (bad_set) are
    refusals whatever the rows"""
    cases = transcript['cases']
    got = harness([(MODEL_FEAT[c['model']], c['prec'] == 'fp64', c['copy'], c['copy'], c['verbs']) for c in cases])
    assert len(cases) > 900
    for c, g in zip(cases, got):
        assert len(g) == len(c['log'])
        for i, ((ok, bits, _, _), rec) in enumerate(zip(g, c['log'])):
            where = (c['model'], c['prec'], c['verbs'], i)
            assert bits == rec[2], where
            assert ok == rec[0], (where, rec[1])


def _closed(have):
    """every present block has what it needs at set (the links a launch lends are lent again at the next launch)"""
    for b in range(6):   # R_BPOS .. R_CT: needs at set; R_CENV needs nothing, R_APP needs contact rows at extended launches only
        need = {1: 0, 2: 1, 3: 2, 4: 3}.get(b)
        if need is not None and (have >> b) & 1 and not (have >> need) & 1:
            return False
    return True


def test_every_sequence_keeps_what_each_block_needs(harness):
    """exhaustively over the verbs that change rows, up to length 4: after every verb each present block has the blocks it needs, and every lent
    block is present"""
    verbs = ('set_bpos', 'clear_bpos', 'set_act', 'clear_act', 'set_mech', 'clear_mech', 'set_ct', 'clear_ct', 'app_on', 'app_off', 'set_sn',
             'clear_sn', 'set_model_rows', 'trace_on', 'trace_off', 'cl_on', 'cl_off', 'aux_on', 'step', 'forward')
    seqs = [s for k in range(1, 5) for s in itertools.product(verbs, repeat=k)]
    for feat, dbl in ((4, 0), (5, 1)):
        for s, g in zip(seqs, harness([(feat, dbl, 0, 0, s) for s in seqs])):
            for i, (_, _, have, lent) in enumerate(g):
                assert _closed(have), (s, i, have)
                assert lent & ~have == 0, (s, i, have, lent)


@pytest.mark.parametrize('verb,clear', [('set_bpos', 'clear_bpos'), ('set_act', 'clear_act'), ('set_mech', 'clear_mech'), ('set_ct', 'clear_ct'),
                                        ('app_on', 'app_off'), ('set_sn', 'clear_sn'), ('trace_on', 'trace_off'), ('cl_on', 'cl_off')])
def test_set_then_clear_restores_the_rows_before(harness, verb, clear):
    """back to the instances that ran before: from every state three verbs reach, set X then clear X restores the exact prior rows and lent bits,
    except where X was already present (its clear then goes further than the set), where the batch's state refuses the set, and for a trace or
    contact lists over the caller's applied rows: the contact rows they lend stay with the applied rows, which hold them at extended launches"""
    verbs = ('set_bpos', 'set_act', 'set_mech', 'set_ct', 'app_on', 'set_sn', 'set_model_rows', 'trace_on', 'cl_on', 'step')
    bit = {'set_bpos': 1, 'set_act': 2, 'set_mech': 3, 'set_ct': 4, 'app_on': 5, 'trace_on': 6, 'cl_on': 7, 'set_sn': 8}[verb]
    pre = [s for k in range(0, 4) for s in itertools.product(verbs, repeat=k)]
    res = harness([(4, 0, 0, 0, s + (verb, clear)) for s in pre])
    checked = 0
    for s, g in zip(pre, res):
        before = (0, 0) if not s else g[len(s) - 1][2:]
        set_ok = g[len(s)][0]
        if (before[0] >> bit) & 1 or not set_ok or (bit in (6, 7) and (before[0] >> 5) & 1):
            continue
        checked += 1
        assert g[len(s) + 1][2:] == before, (s, before, g[len(s) + 1])
    assert checked > 50
