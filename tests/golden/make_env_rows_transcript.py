"""Writes env_rows_transcript.json.gz: verb sequences played on fresh small batches, and what the batch did after every verb.  The committed
transcript was recorded at commit 21bc311 (the per-environment row blocks' lending held by six hand-kept flags) on one H100; the script uses
only API that commit has, so it runs unchanged against it and against later builds.

After every verb a record holds: accepted or refused, the error text of a refusal, a bit per device row pointer of ROWS that is non-null, and,
after launch verbs, a digest of qpos, qvel and obs.  The digest catches rows no pointer shows (body offsets, constant rows) and a launch that ran
another kernel instance.  The sequences: every ordered pair of VERBS on cassie.xml fp32, then N_RANDOM seeded random sequences of SEQ_LEN verbs
over cassie.xml fp32 and cassie_tray_box.xml fp32 / fp64.  Between the two, COPY_CASES: sequences on the batch of a
cassie_sim_t, copied with cassie_sim_copy into a fresh one, whose rows are recorded, then its forward.

    python tests/golden/make_env_rows_transcript.py OUT.json.gz [n_random]      (on a GPU; tests/test_gpu_env_rows.py replays it)
"""
import ctypes as C
import gzip
import hashlib
import importlib
import json
import os
import sys
import time

import numpy as np

REPO = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
ROWS = ('actuators', 'mechanics', 'contact', 'applied', 'trace', 'contacts', 'sensors')
CONFIGS = (('cassie', 'fp32'), ('cassie_tray_box', 'fp32'), ('cassie_tray_box', 'fp64'))
N_ENV = 4
SEQ_LEN = 12
N_RANDOM = 10642   # random sequences: the whole transcript replays in about a minute on an H100
VERBS = ('set_bpos', 'clear_bpos', 'set_act', 'clear_act', 'set_mech', 'clear_mech', 'set_ct', 'set_ct_null', 'clear_ct', 'set_app',
         'app_on', 'app_off', 'set_sn', 'clear_sn', 'set_model_rows', 'get_model_rows', 'trace_on', 'trace_off', 'cl_on', 'cl_off', 'aux_on',
         'aux_off', 'step', 'forward', 'set_const', 'forward_where', 'get_state', 'set_state', 'bad_set')
LAUNCHES = ('step', 'forward', 'set_const', 'forward_where', 'set_state')
COPY_CASES = (('set_ct',), ('set_act', 'set_ct', 'clear_ct'), ('set_mech',), ('set_bpos', 'set_mech'), ('set_ct', 'set_mech', 'clear_ct'),
              ('set_app', 'set_ct'), ('set_sn',), ('set_sn', 'set_act'), ('set_model_rows', 'set_act'), ('set_bpos',), ('set_mech', 'set_bpos', 'clear_mech'),
              ('set_ct_null', 'set_act', 'set_app'))


def package():
    for p in (REPO, os.path.join(REPO, 'tests')):
        if p not in sys.path:
            sys.path.insert(0, p)
    return importlib.import_module('cassie-mujoco-sim_b200')


def digest(b):
    h = hashlib.sha256()
    for a in (b.qpos(), b.qvel(), b.obs()):
        h.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
    return h.hexdigest()[:16]


def pointers(b):
    return ''.join('1' if b.device_ptr(r) else '0' for r in ROWS)


def play(P, b, verb, ctx):
    """one verb on batch b; raises RuntimeError where the library refuses"""
    import torch
    n, e = b.n, min(1, b.n - 1)   # environment e gets its own values (a cassie_sim_t's batch has one)
    one = np.zeros(n, dtype=np.uint8)
    one[e] = 1
    if verb == 'set_bpos':
        pos = b.env_body_pos()
        pos[e, 2, 0] += 0.003
        b.set_env_body_pos(pos)
    elif verb == 'clear_bpos':
        b.clear_env_body_pos()
    elif verb == 'set_act':
        cr, rpm, dl = b.env_actuators()
        b.set_env_actuators(rpm=rpm * 0.97, mask=one)
    elif verb == 'clear_act':
        b.clear_env_actuators()
    elif verb == 'set_mech':
        arm = b.env_mechanics()['armature']
        arm[:, 6:20] *= 1.1
        b.set_env_mechanics(armature=arm, mask=one)
    elif verb == 'clear_mech':
        b.clear_env_mechanics()
    elif verb == 'set_ct':
        solref = b.env_contact()['solref']
        solref[:, :, 0] *= 1.2
        b.set_env_contact(solref=solref, mask=one)
    elif verb == 'set_ct_null':
        b.set_env_contact()
    elif verb == 'clear_ct':
        b.clear_env_contact()
    elif verb == 'set_app':
        xfrc = np.zeros((n, b.L.cassie_batch_nbody(b.h), 6))
        xfrc[e, 1, 2] = 5.0
        b.set_applied_forces(xfrc=xfrc)
    elif verb == 'app_on':
        b.enable_applied_forces(True)
    elif verb == 'app_off':
        b.enable_applied_forces(False)
    elif verb == 'set_sn':
        off = np.zeros((n, 16))
        off[e, 3] = 0.002
        b.set_env_sensors(enc_offset=off)
    elif verb == 'clear_sn':
        b.clear_env_sensors()
    elif verb == 'set_model_rows':
        m = b.get_model('dof_damping')
        m[e, 6] *= 1.05
        b.set_model('dof_damping', m)
    elif verb == 'get_model_rows':
        b.get_model('dof_damping')
    elif verb == 'trace_on':
        b.set_trace([(P.TRACE_QPOS, 2), (P.TRACE_QVEL, 0)], 4)
    elif verb == 'trace_off':
        b.set_trace([])
    elif verb == 'cl_on':
        b.enable_contacts(True)
    elif verb == 'cl_off':
        b.enable_contacts(False)
    elif verb == 'aux_on':
        b.enable_aux(True)
    elif verb == 'aux_off':
        b.enable_aux(False)
    elif verb == 'step':
        b.step(1)
    elif verb == 'forward':
        b.forward()
    elif verb == 'set_const':
        b.set_const()
    elif verb == 'forward_where':
        b.forward_where(torch.tensor(one, device='cuda'))
    elif verb == 'get_state':
        ctx['snap'] = b.get_state(ctx.get('snap'))
    elif verb == 'set_state':
        if 'snap' not in ctx:
            ctx['snap'] = b.get_state()
        b.set_state(ctx['snap'])
    elif verb == 'bad_set':
        b.set_env_actuators(rpm=np.full(b.env_actuators()[1].shape[1], -1.0))
    else:
        raise ValueError(verb)


def record(P, b, verb, ctx):
    try:
        play(P, b, verb, ctx)
        ok, err = True, ''
    except RuntimeError as e:
        ok, err = False, str(e)
    if verb in LAUNCHES:
        b.sync()
    return [ok, err, pointers(b), digest(b) if ok and verb in LAUNCHES else '']


def run_case(P, model, prec, verbs):
    b = P.CassieBatch(N_ENV, modelfile=P.model_path(model), precision=P.FP32 if prec == 'fp32' else P.FP64)
    b.set_pd(P.pd_rows(N_ENV, pTarget=[0.0045, 0, 0.4973, -1.1997, -1.5968] * 2, pGain=[70, 70, 100, 100, 50] * 2, dGain=[7, 7, 8, 8, 5] * 2))
    ctx = {}
    log = [record(P, b, v, ctx) for v in verbs]
    b.close()
    return log


def borrowed(P, h):
    """a CassieBatch over the batch of a cassie_sim_t, which the simulator frees"""
    class Borrowed(P.CassieBatch):
        def close(self):
            self.h = None
    b = Borrowed.__new__(Borrowed)
    b.L, b.n, b.h, b.device = P.lib(), 1, h, 0
    b.nq, b.nv = b.L.cassie_batch_nq(h), b.L.cassie_batch_nv(h)
    b.precision = P.FP64
    return b


def sim_batch(P, sim):
    L = P.lib()
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    return borrowed(P, L.cassie_sim_batch(sim.c))


def run_copy_case(P, verbs):
    src, dst = P.CassieSim(P.model_path('cassie')), P.CassieSim(P.model_path('cassie'))
    sb, db = sim_batch(P, src), sim_batch(P, dst)
    ctx = {}
    log = [record(P, sb, v, ctx) for v in verbs]
    dst.copy(src)
    log.append([True, '', pointers(db), ''])
    log.append(record(P, db, 'forward', ctx))
    return log


def main(path, n_random):
    P = package()
    out = []
    t0 = time.monotonic()
    for a in VERBS:
        for b in VERBS:
            out.append({'model': 'cassie', 'prec': 'fp32', 'verbs': [a, b], 'copy': False, 'log': run_case(P, 'cassie', 'fp32', (a, b))})
    for c in COPY_CASES:
        out.append({'model': 'cassie', 'prec': 'fp64', 'verbs': list(c), 'copy': True, 'log': run_copy_case(P, c)})
    rng = np.random.default_rng(21)
    for i in range(n_random):
        model, prec = CONFIGS[i % len(CONFIGS)]
        verbs = [VERBS[k] for k in rng.integers(0, len(VERBS), SEQ_LEN)]
        out.append({'model': model, 'prec': prec, 'verbs': verbs, 'copy': False, 'log': run_case(P, model, prec, verbs)})
    with gzip.open(path, 'wt') as f:
        json.dump({'n_env': N_ENV, 'rows': ROWS, 'cases': out}, f, separators=(',', ':'))
    print('%d cases in %.1f s' % (len(out), time.monotonic() - t0))


if __name__ == '__main__':
    main(sys.argv[1], int(sys.argv[2]) if len(sys.argv) > 2 else N_RANDOM)
