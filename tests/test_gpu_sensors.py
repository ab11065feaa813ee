"""GPU: sensor models (cassie_batch_set_env_sensors, the F_SN instances): the zero model against the applied-force instances they are the twins of, the
draws recovered from the measurements, their statistics, bias and mount, the generator's counter, parity with the fp64 oracle given the same model
(tests/sensor_support.py), the refusals, the device rows and cassie_sim_copy."""
import ctypes as C
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN, PD_DGAIN, PD_PGAIN, PD_TARGET, REPO, product
import sensor_support as S

pytestmark = pytest.mark.gpu

OB_MPOS, OB_MVEL, OB_JPOS, OB_QUAT, OB_GYRO, OB_ACCEL = 0, 10, 30, 42, 46, 49   # devmodel.h


@pytest.fixture(scope='module')
def P():
    return product()


def _pd(P, b):
    b.set_pd(P.pd_rows(b.n, pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN))


def _pin(P, n):
    pd = P.pd_in_t()
    for side, leg in enumerate((pd.leftLeg, pd.rightLeg)):
        for i in range(5):
            leg.motorPd.pTarget[i], leg.motorPd.pGain[i], leg.motorPd.dGain[i] = PD_TARGET[5 * side + i], PD_PGAIN[i], PD_DGAIN[i]
    return (P.pd_in_t * n)(*[pd] * n)


def _state_out(ys):
    return np.array([np.frombuffer(bytes(y), dtype=np.uint8) for y in ys])


# the batch set-ups that run each F_SN instance (and, with zero applied-force rows instead of sensor rows, its F_XF counterpart)
SETUPS = {
    'f02404': ('cassie', 'FP32', []), 'f22404': ('cassie', 'FP32', ['est']), 'f127c4': ('cassie', 'FP32', ['aux']),
    'f127d7': ('cassie', 'FP32', ['aux', 'acc']), 'd127d7': ('cassie', 'FP64', []),
    'f127df': ('cassie', 'FP32', ['aux', 'acc', 'floor']), 'd127df': ('cassie', 'FP64', ['floor']),
    'f127ff': ('cassie_hfield', 'FP32', ['aux', 'acc', 'terrain']), 'd127ff': ('cassie_hfield', 'FP64', ['terrain']),
}


def _batch(P, tag, n, rows):
    model, prec, extra = SETUPS[tag]
    b = P.CassieBatch(n, modelfile=P.model_path(model), precision=getattr(P, prec))
    if 'est' in extra:
        b.enable_estimator_device()
    if 'aux' in extra:
        b.enable_aux()
    if 'acc' in extra:
        b.enable_accelerations()
    if 'floor' in extra:
        b.set_env_geom_pose('floor', quat=np.array([np.cos(0.005), np.sin(0.005), 0.0, 0.0]))
    if 'terrain' in extra:
        b.set_env_hfield(terrain=0)
    if rows:
        b.set_env_sensors(imu_quat=[1.0, 0, 0, 0])   # the zero model
        b.seed_sensors(12345)
    else:
        b.enable_applied_forces()
    _pd(P, b)
    b.reset()
    return b


# ------------------------------------------------------------------ (a) the zero model is the parent instance
@pytest.mark.parametrize('tag', sorted(SETUPS))
def test_zero_model_is_bitwise_the_parent(P, tag):
    """zero rows, identity mount: qpos, qvel, the observation and the state_out_t of cassie_sim_step_pd_batch equal the F_XF counterpart's bitwise over 200
    ticks (100 compact ticks in launches of 1 and 10, then 100 through the AoS entry point, which also runs the estimator)"""
    n = 64
    a, b = _batch(P, tag, n, False), _batch(P, tag, n, True)
    for k in range(20):
        for x in (a, b):
            x.step(1 if k < 10 else 10)
        assert np.array_equal(a.qpos(), b.qpos()) and np.array_equal(a.qvel(), b.qvel()) and np.array_equal(a.obs(), b.obs()), (tag, k)
    pin = _pin(P, n)
    for k in range(100):
        ya, yb = a.step_pd(pin), b.step_pd(pin)
        assert np.array_equal(_state_out(ya), _state_out(yb)), (tag, k)
    assert np.array_equal(a.qpos(), b.qpos()) and np.array_equal(a.obs(), b.obs()), tag
    assert b.sensor_rng()[1].tolist() == [10 + 10 * 10 + 100] * n   # every step launch advanced the counter by its ticks
    a.close()
    b.close()


# ------------------------------------------------------------------ (b) the draws, recovered on the first tick after a reset
@pytest.mark.parametrize('prec', ['FP32', 'FP64'])
def test_first_tick_draws(P, prec):
    """against a noiseless twin at the same state: the gyro columns differ by numpy's draws (to the rounding of the add), the encoder positions by the
    quantised offset + draw (within one count)"""
    n = 256
    prec_ = getattr(P, prec)
    dt = np.float32 if prec == 'FP32' else np.float64
    a, b = (P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=prec_) for _ in range(2))
    rng = np.random.default_rng(5)
    off, enc_std = rng.uniform(-1e-2, 1e-2, (n, 16)), rng.uniform(0, 5e-3, (n, 16))
    gstd = rng.uniform(0, 0.05, (n, 3))
    imu_noise = np.zeros((n, 9)); imu_noise[:, 3:6] = gstd
    b.set_env_sensors(enc_offset=off, enc_noise=enc_std, imu_noise=imu_noise)
    b.seed_sensors(777)
    a.enable_applied_forces()
    for x in (a, b):
        _pd(P, x)
        x.reset()
    for x in (a, b):
        x.step(1)
    oa, ob = a.obs(), b.obs()
    key, ctr = b.sensor_rng()
    assert key.tolist() == [777 + i for i in range(n)] and ctr.tolist() == [1] * n
    row = b.L.cassie_batch_row_width(b.h, b'sensors')
    assert row == S.SN_W
    rows = np.zeros((n, S.SN_W)); rows[:, 0:16], rows[:, 16:32], rows[:, 32] = off, enc_std, 1.0
    rows[:, 42:45] = gstd
    counts_off = 0
    for e in range(n):
        z = S.draws(777 + e, 0, S.channel_std(rows[e]).astype(dt), dt)
        gyro = (ob[e, OB_GYRO:OB_GYRO + 3] - oa[e, OB_GYRO:OB_GYRO + 3])
        tol = 4 * np.finfo(dt).eps * np.maximum(np.abs(oa[e, OB_GYRO:OB_GYRO + 3]), 1.0)
        assert np.all(np.abs(gyro - z[19:22]) <= tol), (e, gyro, z[19:22])
        # encoders: the drive's count moves by gear (offset + n) / (2 pi / 2^bits), i.e. output radians within one count
        d = np.concatenate([ob[e, OB_MPOS:OB_MPOS + 10] - oa[e, OB_MPOS:OB_MPOS + 10], ob[e, OB_JPOS:OB_JPOS + 6] - oa[e, OB_JPOS:OB_JPOS + 6]])
        want = off[e] + z[:16]
        counts_off = max(counts_off, float(np.abs(d - want).max()))
    # one count: 2 pi / 2^bits over the gear for a drive; the shipped encoders have >= 13 bits and gears >= 16
    assert counts_off <= 2 * np.pi / 2 ** 13 + 1e-6, counts_off
    a.close()
    b.close()


# ------------------------------------------------------------------ (c) statistics
def test_statistics_4096_envs(P):
    """4096 fp32 environments x 100 ticks, gyro noise only, both batches put back at the same snapshot before every tick: per-channel mean and std of
    the measured-minus-true gyro within 3 % of the std, lag-1 and cross-channel correlations below 0.02"""
    n, T = 4096, 100
    sig = np.array([0.01, 0.02, 0.04])
    a, b = (P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32) for _ in range(2))
    noise = np.zeros(9); noise[3:6] = sig
    b.set_env_sensors(imu_noise=noise)
    b.seed_sensors(2024)
    a.enable_applied_forces()
    for x in (a, b):
        _pd(P, x)
        x.reset()
    snap = a.get_state()
    d = np.zeros((T, n, 3))
    for t in range(T):
        for x in (a, b):
            x.set_state(snap)
            x.step(1)
        d[t] = b.obs()[:, OB_GYRO:OB_GYRO + 3] - a.obs()[:, OB_GYRO:OB_GYRO + 3]
    z = d / sig
    m, s = z.mean(axis=(0, 1)), z.std(axis=(0, 1))
    print('mean', m, 'std', s)
    assert np.all(np.abs(m) < 0.03) and np.all(np.abs(s - 1) < 0.03), (m, s)
    lag = [np.corrcoef(z[1:, :, c].ravel(), z[:-1, :, c].ravel())[0, 1] for c in range(3)]
    cross = [np.corrcoef(z[:, :, i].ravel(), z[:, :, j].ravel())[0, 1] for i, j in ((0, 1), (0, 2), (1, 2))]
    envs = np.corrcoef(z[:, 0, 0], z[:, 1, 0])[0, 1]
    print('lag-1', lag, 'cross', cross, 'neighbour envs', envs)
    assert max(abs(v) for v in lag + cross) < 0.02, (lag, cross)
    a.close()
    b.close()


# ------------------------------------------------------------------ (d) bias and mount
@pytest.mark.parametrize('prec', ['FP32', 'FP64'])
def test_bias_and_mount(P, prec):
    """zero std: the orientation is q (x) q_m and the gyro R_m' w + b (accelerometer likewise), against a noiseless twin at the same state, to 1e-6"""
    n = 32
    a, b = (P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=getattr(P, prec)) for _ in range(2))
    rng = np.random.default_rng(8)
    q = rng.normal(size=(n, 4)); q[:, 0] += 4
    bias = rng.uniform(-0.1, 0.1, (n, 6))
    b.set_env_sensors(imu_quat=q, imu_bias=bias)
    a.enable_applied_forces()
    for x in (a, b):
        _pd(P, x)
        x.reset()
    for k in range(30):
        for x in (a, b):
            x.step(1)
        oa, ob = a.obs(), b.obs()
        rows = b.env_sensors()
        for e in range(n):
            qm = rows['imu_quat'][e]
            assert abs(np.linalg.norm(qm) - 1) < 1e-6
            R = S.quat2mat(qm)
            want_q = S._qmul(oa[e, OB_QUAT:OB_QUAT + 4], qm)
            assert np.abs(ob[e, OB_QUAT:OB_QUAT + 4] - want_q).max() < 1e-6
            assert np.abs(ob[e, OB_GYRO:OB_GYRO + 3] - (R.T @ oa[e, OB_GYRO:OB_GYRO + 3] + bias[e, :3])).max() < 1e-6 * max(1.0, np.abs(oa[e, OB_GYRO:OB_GYRO + 3]).max())
            assert np.abs(ob[e, OB_ACCEL:OB_ACCEL + 3] - (R.T @ oa[e, OB_ACCEL:OB_ACCEL + 3] + bias[e, 3:])).max() < 1e-6 * max(1.0, np.abs(oa[e, OB_ACCEL:OB_ACCEL + 3]).max())
        # the motor PD reads the encoders only (no estimator here), so the mounted IMU leaves the motion alone
        assert np.array_equal(a.qpos(), b.qpos())
    a.close()
    b.close()


# ------------------------------------------------------------------ (e) reproducibility and counter semantics
def _noisy(P, n, prec=None, seed=11):
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=prec or P.FP32)
    b.set_env_sensors(enc_noise=np.full(16, 2e-4), imu_noise=[1e-3] * 3 + [5e-4] * 3 + [1e-2] * 3)
    b.seed_sensors(seed)
    _pd(P, b)
    b.reset()
    return b


def test_reproducibility_and_counter(P):
    """equal keys and counters give bitwise-equal trajectories, different keys do not; a snapshot restore with the counter restored continues bitwise;
    a reset does not replay; a 50-tick launch advances the counter by 50 and a forward launch not at all"""
    import torch
    n = 128
    a, b, c = _noisy(P, n), _noisy(P, n), _noisy(P, n, seed=12)
    for x in (a, b, c):
        x.enable_estimator_device()
        x.step(50)
    assert np.array_equal(a.obs(), b.obs()) and np.array_equal(a.qpos(), b.qpos())
    assert not np.array_equal(a.obs(), c.obs())
    assert a.sensor_rng()[1].tolist() == [50] * n
    a.forward()
    assert a.sensor_rng()[1].tolist() == [50] * n
    # snapshot + counter restore
    snap = a.get_state()
    a.sync()
    rng_rows = a.torch_view('sensor_rng').clone()
    a.step(30)
    q1, o1 = a.qpos(), a.obs()
    a.set_state(snap)
    a.torch_view('sensor_rng').copy_(rng_rows)
    torch.cuda.synchronize()
    a.step(30)
    assert np.array_equal(a.qpos(), q1) and np.array_equal(a.obs(), o1)
    # without the counter restore the same snapshot draws new noise
    a.set_state(snap)
    a.step(30)
    assert not np.array_equal(a.obs(), o1)
    # a reset keeps the counter: the first ticks of two episodes differ
    d = _noisy(P, n)
    d.step(1)
    first = d.obs()
    d.reset()
    d.step(1)
    assert d.sensor_rng()[1].tolist() == [2] * n and not np.array_equal(d.obs()[:, OB_GYRO:OB_GYRO + 6], first[:, OB_GYRO:OB_GYRO + 6])
    for x in (a, b, c, d):
        x.close()


# ------------------------------------------------------------------ (f) parity with the oracle
def test_parity_with_the_oracle(P, oracle_mod):
    """the same model in front of the fp64 oracle: fp64 chain twin standing, estimator on (qpos within 1e-9, the state_out_t pelvis and feet within 1e-6),
    and fp32 plain twin on bench config 3's push (within config 3's bars)"""
    sys.path.insert(0, REPO)
    import bench
    from test_gpu_configs import BARS
    O = oracle_mod
    n = 4
    row = S.make_row(enc_offset=np.linspace(-1e-3, 1e-3, 16), enc_noise=np.full(16, 2e-4), imu_quat=[1, 0.01, -0.02, 0.005], imu_bias=[0.01, -0.01, 0.005, 0.02, -0.03, 0.01],
                     imu_noise=[1e-3] * 3 + [5e-4] * 3 + [1e-2] * 3)
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP64)
    b.set_env_sensors(**{k: np.asarray(v) for k, v in S.row_args(row).items()})
    b.seed_sensors(99)
    _pd(P, b)
    b.reset()
    pin = _pin(P, n)
    os_ = [O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel')) for _ in range(n)]
    ms = [S.OracleSensors(o, 'cassie', row, 99 + e, 0) for e, o in enumerate(os_)]
    u = O.make_pd(pTarget=PD_TARGET, pGain=PD_PGAIN, dGain=PD_DGAIN)
    y = P.state_out_t()
    worst_q, worst_y = 0.0, 0.0
    for t in range(300):
        ys = b.step_pd(pin)
        for e, (o, m) in enumerate(zip(os_, ms)):
            m.step_pd(u, y)
            if e == 2:
                worst_y = max(worst_y, float(np.abs(np.array(ys[e].pelvis.orientation[:]) * np.sign(ys[e].pelvis.orientation[0]) - np.array(y.pelvis.orientation[:]) * np.sign(y.pelvis.orientation[0])).max()),
                              float(np.abs(np.array(ys[e].leftFoot.position[:]) - np.array(y.leftFoot.position[:])).max()))
        worst_q = max(worst_q, max(float(np.abs(b.qpos()[e] - o.arr('qpos')).max()) for e, o in enumerate(os_)))
    print('fp64 chain twin: qpos %.2e state_out %.2e' % (worst_q, worst_y))
    assert worst_q < 1e-9 and worst_y < 1e-6, (worst_q, worst_y)
    b.close()
    # fp32 plain twin, config 3's push
    n, T = 256, 400
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    b.set_env_sensors(**{k: np.asarray(v) for k, v in S.row_args(row).items()})
    b.seed_sensors(99)
    _pd(P, b)
    b.reset()
    q0 = b.qpos()
    push = bench.philox_uniform(1234, 0, (n, 2), -100.0, 100.0)
    xf = np.zeros((n, b.L.cassie_batch_nbody(b.h), 6))
    xf[:, 1, :2] = push
    b.set_applied_forces(xfrc=xf)
    b.step(100)
    b.set_applied_forces(xfrc=np.zeros_like(xf))
    b.step(T - 100)
    got = b.qpos()
    sample = [3, 77, 150, 255]
    err = []
    for e in sample:
        o = O.OracleSim(os.path.join(GOLDEN, 'cassie.omodel'))
        o.arr('qpos')[:o.nq] = q0[e]
        o.forward()
        m = S.OracleSensors(o, 'cassie', row, 99 + e, 0)
        o.arr('xfrc_applied').reshape(-1, 6)[1, :2] = push[e]
        for t in range(T):
            if t == 100:
                o.arr('xfrc_applied')[:] = 0
            m.step_pd(u)
        err.append(float(np.abs(got[e] - o.arr('qpos')[:o.nq]).max()))
    print('fp32 plain twin, config 3 push: %s' % err)
    assert max(err) <= BARS[3][2], err
    b.close()


# ------------------------------------------------------------------ (g) refusals
def test_refusals(P):
    n = 4
    b = P.CassieBatch(n, modelfile=P.model_path('cassie'), precision=P.FP32)
    bad = [dict(enc_offset=np.where(np.arange(16) == 3, np.nan, 0.0)), dict(enc_noise=-np.ones(16) * 1e-3), dict(imu_quat=[0, 0, 0, 0]),
           dict(imu_bias=[0, 0, np.inf, 0, 0, 0]), dict(imu_noise=[0, 0, 0, 0, -1, 0, 0, 0, 0])]
    for kw in bad:
        with pytest.raises(RuntimeError) as ex:
            b.set_env_sensors(**kw)
        assert 'environment 0' in str(ex.value), str(ex.value)
    assert b.device_ptr('sensors') in (None, 0)   # nothing was allocated
    with pytest.raises(RuntimeError):
        b.seed_sensors(1)
    b.set_env_sensors(enc_noise=np.full(16, 1e-4))
    with pytest.raises(RuntimeError, match='sensor models'):
        b.enable_contacts(True)
    with pytest.raises(RuntimeError, match='sensor models'):
        b.set_trace([(0, 0)], 4)
    b.clear_env_sensors()
    b.enable_contacts(True)
    with pytest.raises(RuntimeError, match='contact lists'):
        b.set_env_sensors(enc_noise=np.full(16, 1e-4))
    b.enable_contacts(False)
    b.set_trace([(0, 0)], 4)
    with pytest.raises(RuntimeError, match='trace'):
        b.set_env_sensors(enc_noise=np.full(16, 1e-4))
    b.close()


# ------------------------------------------------------------------ (h) device rows and cassie_sim_copy
def test_device_rows_and_copy(P):
    """a write through torch_view('sensors') takes effect at the next launch (equal to the verb's write); cassie_sim_copy copies rows and generator"""
    import torch
    n = 64
    a, b = _noisy(P, n), _noisy(P, n)
    for x in (a, b):
        x.set_stream(torch.cuda.current_stream().cuda_stream)
    v = a.torch_view('sensors')
    assert v.shape == (n, S.SN_W)
    v[:, S.SN_GYRO_BIAS:S.SN_GYRO_BIAS + 3] = 0.25
    bias = np.zeros(6); bias[:3] = 0.25
    b.set_env_sensors(imu_bias=bias)
    for x in (a, b):
        x.step(20)
    assert np.array_equal(a.obs(), b.obs()) and np.array_equal(a.qpos(), b.qpos())
    assert np.allclose(a.env_sensors()['imu_bias'][:, :3], 0.25)
    # legacy simulators: cassie_sim_copy copies the rows and the generator, so the copy draws what the original does
    s = P.CassieSim(P.model_path('cassie'))
    L = P.lib()
    L.cassie_sim_batch.restype = C.c_void_p
    L.cassie_sim_batch.argtypes = [C.c_void_p]
    sb = L.cassie_sim_batch(s.c)
    L.cassie_batch_set_env_sensors.argtypes = [C.c_void_p] * 7
    noise = np.array([1e-3] * 3 + [5e-4] * 3 + [1e-2] * 3)
    assert L.cassie_batch_set_env_sensors(sb, None, None, None, None, noise.ctypes.data, None) == 0
    pd = _pin(P, 1)[0]
    for _ in range(10):
        s.step_pd(pd)
    d = s.duplicate()
    for _ in range(40):
        s.step_pd(pd)
        d.step_pd(pd)
    assert np.array_equal(s.qpos(), d.qpos())
    a.close()
    b.close()
