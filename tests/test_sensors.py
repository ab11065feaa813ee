"""Sensor models (cassie_batch_set_env_sensors): the generator and the draw against numpy, and the product's stepper source in the host emulation, with
the encoders, the IMU mount, bias and noise applied to what the controller stage measures (the F_SN instances), against the fp64 oracle with the same
model in front of its controller stage (tests/sensor_support.py).  The GPU twins are in tests/test_gpu_sensors.py.

The emulation is tests/emu/emu_sensors.cpp: the chain-twin source (extended, with model-valued applied, contact, mechanics, actuator and offset rows)
and the plain-twin source (the plain kind, its scratch tail NaN-poisoned), and their F_XF parents."""
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO
import sensor_support as S

sys.path.insert(0, REPO)
import bench  # noqa: E402

MODELS = os.path.join(REPO, 'cassie-mujoco-sim_b200', 'models')
PD_ROW = np.concatenate([np.zeros(10), PD_TARGET, np.zeros(10), PD_PGAIN, PD_DGAIN])
OB_MPOS, OB_JPOS, OB_QUAT, OB_GYRO, OB_ACCEL, OB_MAG = 0, 30, 42, 46, 49, 52   # devmodel.h


def noisy_row(seed=0):
    """a model with every part on: the model files' noise= values (shin / tarsus 2e-4, gyro 5e-4, accelerometer 1e-2) and more, offsets, a tilted mount"""
    rng = np.random.default_rng(seed)
    enc_noise = np.full(16, 1e-4)
    enc_noise[10:] = 2e-4
    q = np.array([1.0, 0.02, -0.015, 0.01])
    return S.make_row(enc_offset=rng.uniform(-2e-3, 2e-3, 16), enc_noise=enc_noise, imu_quat=q, imu_bias=np.concatenate([rng.uniform(-0.01, 0.01, 3), rng.uniform(-0.05, 0.05, 3)]),
                      imu_noise=np.array([1e-3, 1e-3, 1e-3, 5e-4, 5e-4, 5e-4, 1e-2, 1e-2, 1e-2]))


# ------------------------------------------------------------------ 1. the generator
def test_generator_matches_numpy():
    """Philox-4x64-10 of the kernel source (through the emulation) and of the oracle-side restatement equal numpy's Philox bitwise over 1e5 random
    (t, j, key), the counter's low word and the key spanning all 64 bits"""
    rng = np.random.default_rng(3)
    n = 100_000
    t = rng.integers(0, 2 ** 64 - 1, n, dtype=np.uint64, endpoint=True)
    t[:8] = [0, 1, 2, 2 ** 32 - 1, 2 ** 32, 2 ** 63, 2 ** 64 - 2, 2 ** 64 - 1]
    j = rng.integers(0, 7, n, dtype=np.uint64)
    j[:8] = 0
    key = rng.integers(0, 2 ** 64 - 1, n, dtype=np.uint64, endpoint=True)
    want = np.array([S.numpy_block(t[i], j[i], key[i]) for i in range(n)], dtype=np.uint64)
    assert np.array_equal(S.emu_philox(t, j, key), want)
    assert np.array_equal(S.philox(t, j, key), want)


def test_draws_match_numpy():
    """n = fl(fl(std C) x) in the emulation equals numpy's in fp32 and fp64 bitwise; x is the exact Irwin-Hall integer, within +-131070"""
    rng = np.random.default_rng(4)
    w = rng.integers(0, 2 ** 64 - 1, 200_000, dtype=np.uint64, endpoint=True)
    w[:4] = [0, 2 ** 64 - 1, 0x7fff7fff7fff7fff, 0x8000800080008000]
    sigma = np.exp(rng.uniform(np.log(1e-6), np.log(10.0), w.size))
    sigma[:8] = 0.0
    o32, o64 = S.emu_noise(sigma, w)
    assert np.array_equal(o32.view(np.uint32), S.noise(sigma, w, np.float32).view(np.uint32))
    assert np.array_equal(o64.view(np.uint64), S.noise(sigma, w, np.float64).view(np.uint64))
    x = S.irwin_hall(w)
    assert x[0] == -131070 and x[1] == 131070 and x[2] == -2 and x[3] == 2
    # the draw's moments: zero mean, unit variance, kurtosis 2.7 (Irwin-Hall of four), tails cut at sqrt(12) std
    z = x * S.C_NOISE
    assert abs(z.mean()) < 0.01 and abs(z.std() - 1) < 0.01 and abs(np.mean(z ** 4) / np.mean(z ** 2) ** 2 - 2.7) < 0.03 and np.abs(z).max() <= np.sqrt(12)


# ------------------------------------------------------------------ 2. against the oracle with the same model
def _run_pair(oracle_mod, model, mode, fp32, ticks, push):
    o = oracle_mod.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    o.set_caps()
    e = S.SnSim(os.path.join(MODELS, model + '.cmodel'), mode, fp32)
    row, key, ctr = noisy_row(1), 0x1234_5678_9abc_def0, 2 ** 32 - 20   # the counter crosses its low word
    e.set_row(row, key, ctr)
    m = S.OracleSensors(o, model, row, key, ctr)
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    nq = o.nq
    worst_q, worst_imu, worst_acc = 0.0, 0.0, 0.0
    for t in range(ticks):
        if push and t == 0:
            p = bench.philox_uniform(1234, 0, (bench.CONFIGS[3]['envs'], 2), -100.0, 100.0)[7]
            o.arr('xfrc_applied').reshape(-1, 6)[1, :2] = p
            x = np.zeros(8); x[:2] = p; x[6] = 1
            e.L.emu_set(e.h, b'xfrc', S._dp(x), 8)
        elif push and t == 100:
            o.arr('xfrc_applied')[:] = 0
            e.L.emu_set(e.h, b'xfrc', S._dp(np.zeros(8)), 8)
        meas = m.measure_now()
        m.step_pd(u)
        e.step(PD_ROW)
        obs = e.get('obs')
        worst_q = max(worst_q, float(np.abs(e.get('qpos')[:nq] - o.arr('qpos')[:nq]).max()))
        imu = np.concatenate([obs[OB_QUAT:OB_QUAT + 4] * np.sign(obs[OB_QUAT]), obs[OB_GYRO:OB_GYRO + 3]])
        worst_imu = max(worst_imu, float(np.abs(imu - np.concatenate([meas[16:20] * np.sign(meas[16]), meas[20:23]])).max()))
        worst_acc = max(worst_acc, float(np.abs(obs[OB_ACCEL:OB_ACCEL + 6] - meas[23:29]).max()))
    assert e.counter() == ctr + ticks
    e.close()
    return o, worst_q, worst_imu, worst_acc


@pytest.mark.parametrize('push', [False, True], ids=['stand', 'push'])
@pytest.mark.parametrize('mode', [S.CHAIN, S.PLAIN], ids=['chain', 'plain'])
def test_sensor_model_follows_the_oracle(oracle_mod, mode, push):
    """fp64, 500 ticks standing under PD, or bench config 3's push for 100 of 400 ticks: qpos within 1e-9 of the oracle whose controller stage
    measures through the same model, seed and counter; the IMU columns of the observation are the restated measurement (1e-9)"""
    model = bench.CONFIGS[3]['model'] if push else 'cassie'
    o, wq, wi, wa = _run_pair(oracle_mod, model, mode, False, 400 if push else 500, push)
    print(model, mode, push, 'qpos %.2e orientation / gyro %.2e accelerometer / magnetometer %.2e' % (wq, wi, wa))
    assert wq < 1e-9 and wi < 1e-9 and wa < 1e-9, (wq, wi, wa)
    # the model changes the motion
    o0 = oracle_mod.OracleSim(os.path.join(GOLDEN, model + '.omodel'))
    o0.set_caps()
    if push:
        o0.arr('xfrc_applied').reshape(-1, 6)[1, :2] = bench.philox_uniform(1234, 0, (bench.CONFIGS[3]['envs'], 2), -100.0, 100.0)[7]
    u = oracle_mod.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    for t in range(400 if push else 500):
        if push and t == 100:
            o0.arr('xfrc_applied')[:] = 0
        o0.step_pd(u)
    assert np.abs(o0.arr('qpos') - o.arr('qpos')).max() > 1e-5
    o.close()
    o0.close()


def test_fp32_plain_twin_follows_the_oracle(oracle_mod):
    """the fp32 plain twin (what the headline workload runs with sensor rows) on config 3's push: qpos within 1e-4 of the fp64 oracle over 400 ticks,
    the tolerance of the fp32 configuration parity; orientation and gyro within 3e-3 of the fp64 measurement through the same model (the rates and
    accelerations under the push are the fp32 physics', so the accelerometer is left to the fp64 cases)"""
    o, wq, wi, wa = _run_pair(oracle_mod, bench.CONFIGS[3]['model'], S.PLAIN, True, 400, True)
    print('fp32 plain qpos %.2e orientation / gyro %.2e accelerometer / magnetometer %.2e' % (wq, wi, wa))
    assert wq < 1e-4 and wi < 3e-3, (wq, wi)
    o.close()


# ------------------------------------------------------------------ 3. the zero model is the parent instance
@pytest.mark.parametrize('fp32', [False, True], ids=['fp64', 'fp32'])
@pytest.mark.parametrize('pair', [(S.CHAIN_PARENT, S.CHAIN), (S.PLAIN_PARENT, S.PLAIN)], ids=['chain', 'plain'])
def test_zero_model_is_bitwise_the_parent(pair, fp32):
    """zero rows with the identity mount, any key and counter: qpos, qvel, the observation (the estimator's columns included on the chain twin), the
    controller state and the FIR taps equal the F_XF parent's bitwise over 300 ticks, in launches of 1 and 7 ticks"""
    a, b = (S.SnSim(os.path.join(MODELS, 'cassie.cmodel'), m, fp32) for m in pair)
    b.set_row(S.make_row(), key=987654321, counter=5)
    if pair[1] == S.CHAIN:
        a.enable_est()
        b.enable_est()
    for k in range(60):
        n = 1 if k < 20 else 7
        a.step(PD_ROW, n)
        b.step(PD_ROW, n)
        for f in ('qpos', 'qvel', 'obs', 'cst', 'dfilt'):
            assert np.array_equal(a.get(f), b.get(f)), (k, f)
    assert b.counter() == 5 + 20 + 40 * 7
    a.close()
    b.close()
