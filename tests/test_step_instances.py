"""The step-kernel instance table (csrc/step_instances.inc) and the rule that picks a launch's instance from it (csrc/step_select.h), compiled on
the host with g++ (no GPU, no CUDA headers).

tests/golden/step_instance_routes.npz holds the instance every request ran when each feature's instances were routed by hand-written branches
(tests/golden/make_step_instance_routes.py).  The rule must reproduce it except on two requests no batch can make: F_TC | F_CL (set_trace and
enable_contacts refuse each other), which the old branches sent to a contact-list instance and the rule to none, and F_SN without F_XF (a batch
with sensor rows gets applied rows before it launches)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import GOLDEN, REPO
from test_env_geom_resources import _build_module

CSRC = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'csrc')
F_XF, F_TC, F_CL, F_SN = 1024, 2048, 4096, 8192
NBITS = 14

HARNESS = r'''
#include <cstdio>
#include "step_select.h"
using namespace cassie;
static const char *TAGS[] = {
#define STEP_INSTANCE(tag) #tag,
#include "step_instances.inc"
#undef STEP_INSTANCE
};
static const StepInstance TABLE[] = {
#define STEP_INSTANCE(tag) step_instance(#tag),
#include "step_instances.inc"
#undef STEP_INSTANCE
};
int main() {
  const int n = sizeof TABLE / sizeof TABLE[0];
  printf("%d\n", n);
  for (int i = 0; i < n; i++) printf("%s %d %d %d\n", TAGS[i], TABLE[i].dbl, TABLE[i].kind, TABLE[i].feat);
  for (int dbl = 0; dbl < 2; dbl++) for (int kind = 0; kind < 3; kind++) for (int f = 0; f < (1 << NBITS); f++) {
    const StepChoice s = step_select(TABLE, n, dbl, kind, f);
    printf("%d %d\n", s.kind, s.index);
  }
}
'''


@pytest.fixture(scope='module')
def compiled(tmp_path_factory):
    """(table: [(tag, dbl, kind, feat)], kind [2, 3, 2^14], index [2, 3, 2^14]) as the compiled header picks them"""
    tmp = tmp_path_factory.mktemp('step_select')
    src, exe = tmp / 'select.cpp', tmp / 'select'
    src.write_text(HARNESS)
    subprocess.check_call(['g++', '-O1', '-std=c++17', '-DNBITS=%d' % NBITS, '-I', CSRC, '-o', str(exe), str(src)])
    lines = subprocess.check_output([str(exe)], text=True).splitlines()
    n = int(lines[0])
    table = [(t, bool(int(d)), int(k), int(f)) for t, d, k, f in (line.split() for line in lines[1:n + 1])]
    routes = np.array([line.split() for line in lines[n + 1:]], dtype=np.int64).reshape(2, 3, 1 << NBITS, 2)
    return table, routes[..., 0], routes[..., 1]


def test_build_lists_the_compiled_table(compiled):
    table, _, _ = compiled
    assert _build_module().STEP_INSTANCES == [(t, 'double' if dbl else 'float', kind, feat) for t, dbl, kind, feat in table]
    assert len({t for t, *_ in table}) == len(table)


def test_routes_match_the_fixture(compiled):
    table, kind, index = compiled
    golden = np.load(os.path.join(GOLDEN, 'step_instance_routes.npz'))
    tags = [t for t, *_ in table]
    want = np.array([tags.index(t) for t in golden['tags']])[golden['instance']]
    want[golden['instance'] < 0] = -1
    bits = np.arange(1 << NBITS)
    both = ((bits & F_TC) != 0) & ((bits & F_CL) != 0)
    sensors_alone = ((bits & F_SN) != 0) & ((bits & F_XF) == 0)
    assert (index[:, :, both] == -1).all()   # a trace and contact lists: no instance
    differ = (kind != golden['kind']) | (index != want)
    differ[:, :, both | sensors_alone] = False
    assert not differ.any(), [('fd'[d], k, hex(b), (golden['kind'][d, k, b], want[d, k, b]), (kind[d, k, b], index[d, k, b])) for d, k, b in np.argwhere(differ)[:10]]


def test_every_instance_is_picked_for_its_own_features(compiled):
    table, kind, index = compiled
    for i, (t, dbl, k, feat) in enumerate(table):
        assert (kind[int(dbl), k, feat], index[int(dbl), k, feat]) == (k, i), t


def test_no_two_covering_instances_tie():
    """for every precision, kind and request, at most one instance of the fewest bits has every requested bit"""
    table = _build_module().STEP_INSTANCES
    bits = np.arange(1 << NBITS)
    for real in ('float', 'double'):
        for k in range(3):
            feats = np.array([f for _, r, kk, f in table if r == real and kk == k])
            covers = (feats[None, :] & bits[:, None]) == bits[:, None]
            size = np.where(covers, np.array([bin(f).count('1') for f in feats])[None, :], 99)
            ties = (size == size.min(axis=1, keepdims=True)) & covers
            assert (ties.sum(axis=1) <= 1).all(), (real, k, [hex(b) for b in bits[ties.sum(axis=1) > 1][:5]])
