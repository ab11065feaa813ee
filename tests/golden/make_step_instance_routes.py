#!/usr/bin/env python3
"""Regenerates tests/golden/step_instance_routes.npz: the step-kernel instance every launch request ran at commit 1128d37, the last one that picked
instances with hand-written branches (step_entry in csrc/cassie_b200.cu).  Needs the repository's git history and g++; the tests use the committed file.

The script takes that commit's step_entry and its entry declarations from `git show`, compiles them on the host with stub entry functions that return
their tag, and runs them with launch_kind's applied-force fallback on every request: kind 0 plain / 1 extended / 2 plain + estimator, any of the 14
feature bits (csrc/devmodel.h F_*), each precision.  The fallback is probed with the whole request; launch_kind probed with the bits a plain batch can
hold (F_ALL | F_EG | F_TR | F_BP | F_XF | F_SN), which is the whole request of every plain launch, as the other bits come with rows that make the
batch extended.

  tags       the 100 instance tags, in the commit's declaration order
  kind       [precision (0 float, 1 double), requested kind, request bits]: the kind the launch ran
  instance   [same]: index into tags, -1 where step_entry returned no instance
"""
import os
import re
import subprocess
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
COMMIT = '1128d37'
NBITS = 14

HARNESS = r'''
#include <cstdio>
#include <type_traits>
#include "devmodel.h"
%(stubs)s
namespace cassie {
%(step_entry)s
template <typename real> void dump() {
  for (int kind = 0; kind < 3; kind++) for (int f = 0; f < (1 << %(nbits)d); f++) {
    int ext = kind;
    if ((f & F_XF) && ext != 1 && !step_entry<real>(ext, f)) ext = 1;   // launch_kind's fallback
    const char *t = (const char *)step_entry<real>(ext, f);
    printf("%%d %%s\n", ext, t ? t : "-");
  }
}
}
int main() { cassie::dump<float>(); cassie::dump<double>(); }
'''


def show(path):
    return subprocess.check_output(['git', '-C', REPO, 'show', '%s:cassie-mujoco-sim_b200/csrc/%s' % (COMMIT, path)], text=True)


def main():
    src = show('cassie_b200.cu')
    decl = re.search(r'#define CASSIE_STEP_ENTRY\(tag\).*?\n(.*?)#undef CASSIE_STEP_ENTRY', src, re.S).group(1)
    tags = re.findall(r'CASSIE_STEP_ENTRY\((\w+)\)', decl)
    a = src.index('template <typename real> static const void *step_entry(')
    step_entry = src[a:src.index('\n}\n', a) + 3]
    stubs = '\n'.join('extern "C" const void *cassie_step_entry_%s(void) { return "%s"; }' % (t, t) for t in tags)
    with tempfile.TemporaryDirectory() as tmp:
        with open(os.path.join(tmp, 'devmodel.h'), 'w') as f:
            f.write(show('devmodel.h'))
        with open(os.path.join(tmp, 'routes.cpp'), 'w') as f:
            f.write(HARNESS % dict(stubs=stubs, step_entry=step_entry, nbits=NBITS))
        exe = os.path.join(tmp, 'routes')
        subprocess.check_call(['g++', '-O1', '-std=c++17', '-I', tmp, '-o', exe, os.path.join(tmp, 'routes.cpp')])
        rows = [line.split() for line in subprocess.check_output([exe], text=True).splitlines()]
    shape = (2, 3, 1 << NBITS)
    kind = np.array([int(k) for k, _ in rows], dtype=np.int8).reshape(shape)
    instance = np.array([tags.index(t) if t != '-' else -1 for _, t in rows], dtype=np.int16).reshape(shape)
    np.savez_compressed(os.path.join(HERE, 'step_instance_routes.npz'), tags=np.array(tags), kind=kind, instance=instance)


if __name__ == '__main__':
    main()
