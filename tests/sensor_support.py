"""The sensor model of the F_SN step-kernel instances (cassie_batch_set_env_sensors), restated in numpy, and the same model put in front of the fp64
oracle's controller stage.  TEST INFRASTRUCTURE ONLY.

The oracle's cassie_sim_step_pd reads last step's sensordata in its controller stage (oracle/cassie_oracle.c sensor_data_) and then steps the physics,
which writes the true sensordata again.  So measuring is: overwrite the oracle's sensordata with the measured values right before step_pd; MuJoCo's own
sensordata is back after the step, as it is in the kernel, which measures a shared-memory copy."""
import ctypes as C
import os
import subprocess

import numpy as np

from mechanics_support import table

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(os.path.dirname(HERE), 'cassie-mujoco-sim_b200', 'csrc')

SN_W, SN_ENC_OFF, SN_ENC_STD, SN_QUAT, SN_ORI_STD, SN_GYRO_BIAS, SN_GYRO_STD, SN_ACC_BIAS, SN_ACC_STD = 52, 0, 16, 32, 36, 39, 42, 45, 48   # devmodel.h
NCH = 25
C_NOISE = 1.0 / np.sqrt((65536.0 ** 2 - 1) / 3)   # the draw's scale; (real) of it in fp32
DRIVE_S = [0, 1, 2, 3, 4, 8, 9, 10, 11, 12]        # sensordata index of drive encoder c
JOINT_S = [5, 6, 7, 13, 14, 15]                    # ... of joint encoder c - 10

M0, M1 = 0xD2E7470EE14C6C93, 0xCA5A826395121157
W0, W1 = 0x9E3779B97F4A7C15, 0xBB67AE8584CAA73B
MASK = (1 << 64) - 1


# ------------------------------------------------------------------ the generator and the draw
def _mulhilo(a, b):
    """uint64 arrays a * b -> (hi, lo), from 32-bit halves (numpy has no 128-bit product)"""
    m32 = np.uint64(0xffffffff)
    a0, a1, b0, b1 = a & m32, a >> np.uint64(32), b & m32, b >> np.uint64(32)
    p00, p01, p10, p11 = a0 * b0, a0 * b1, a1 * b0, a1 * b1
    mid = (p00 >> np.uint64(32)) + (p01 & m32) + (p10 & m32)
    hi = p11 + (p01 >> np.uint64(32)) + (p10 >> np.uint64(32)) + (mid >> np.uint64(32))
    return hi, a * b


def philox(t, j, key):
    """Philox-4x64-10 blocks with counter (t, j, 0, 0) and key (key, 0), vectorised: uint64 arrays -> [..., 4]"""
    with np.errstate(over='ignore'):
        c0, c1 = np.asarray(t, dtype=np.uint64), np.asarray(j, dtype=np.uint64)
        c0, c1 = np.broadcast_arrays(c0, c1)
        c2 = np.zeros_like(c0); c3 = np.zeros_like(c0)
        k0 = np.broadcast_to(np.asarray(key, dtype=np.uint64), c0.shape).copy(); k1 = np.zeros_like(c0)
        for _ in range(10):
            hi0, lo0 = _mulhilo(np.uint64(M0), c0)
            hi1, lo1 = _mulhilo(np.uint64(M1), c2)
            c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
            k0 = k0 + np.uint64(W0); k1 = k1 + np.uint64(W1)
    return np.stack([c0, c1, c2, c3], axis=-1)


def numpy_block(t, j, key):
    """the same block from numpy's own Philox: its counter is incremented before the first output"""
    ctr = (int(t) + (int(j) << 64) - 1) % (1 << 256)
    return np.random.Philox(counter=ctr, key=int(key)).random_raw(4)


def irwin_hall(word):
    """x = u0 + u1 + u2 + u3 - 131070 over the four 16-bit parts of each uint64 word (exact integers)"""
    w = np.asarray(word, dtype=np.uint64)
    return sum(((w >> np.uint64(16 * i)) & np.uint64(0xffff)).astype(np.int64) for i in range(4)) - 131070


def noise(sigma, word, dtype=np.float64):
    """n = fl(fl(sigma C) x) in the given precision"""
    s = np.asarray(sigma, dtype=dtype)
    return (s * dtype(C_NOISE)).astype(dtype) * irwin_hall(word).astype(dtype)


def draws(key, t, sigma, dtype=np.float64):
    """the 25 draws of one tick: channel c = word c % 4 of block (t, c / 4); sigma [25] in channel order"""
    blocks = philox(np.full(7, t, dtype=np.uint64), np.arange(7, dtype=np.uint64), np.uint64(key))
    return noise(sigma, blocks.reshape(-1)[:NCH], dtype)


def channel_std(row):
    """the std of each of the 25 channels, from a sensor row"""
    r = np.asarray(row, dtype=np.float64)
    return np.concatenate([r[SN_ENC_STD:SN_ENC_STD + 16], r[SN_ORI_STD:SN_ORI_STD + 3], r[SN_GYRO_STD:SN_GYRO_STD + 3], r[SN_ACC_STD:SN_ACC_STD + 3]])


def make_row(enc_offset=None, enc_noise=None, imu_quat=(1, 0, 0, 0), imu_bias=None, imu_noise=None):
    """one environment's device row, the verb's argument shapes, the quaternion normalised as the verb does"""
    row = np.zeros(SN_W)
    if enc_offset is not None:
        row[SN_ENC_OFF:SN_ENC_OFF + 16] = enc_offset
    if enc_noise is not None:
        row[SN_ENC_STD:SN_ENC_STD + 16] = enc_noise
    q = np.asarray(imu_quat, dtype=np.float64)
    row[SN_QUAT:SN_QUAT + 4] = q / np.sqrt(np.sum(q * q))
    if imu_bias is not None:
        row[SN_GYRO_BIAS:SN_GYRO_BIAS + 3], row[SN_ACC_BIAS:SN_ACC_BIAS + 3] = imu_bias[:3], imu_bias[3:]
    if imu_noise is not None:
        row[SN_ORI_STD:SN_ORI_STD + 3], row[SN_GYRO_STD:SN_GYRO_STD + 3], row[SN_ACC_STD:SN_ACC_STD + 3] = imu_noise[:3], imu_noise[3:6], imu_noise[6:]
    return row


def row_args(row):
    """the verb's arguments (enc_offset, enc_noise, imu_quat, imu_bias, imu_noise) of a row"""
    r = np.asarray(row)
    return dict(enc_offset=r[0:16], enc_noise=r[16:32], imu_quat=r[32:36], imu_bias=np.concatenate([r[39:42], r[45:48]]),
                imu_noise=np.concatenate([r[36:39], r[42:45], r[48:51]]))


# ------------------------------------------------------------------ the model on a sensordata vector (fp64)
def _qmul(a, b):
    return np.array([a[0] * b[0] - a[1] * b[1] - a[2] * b[2] - a[3] * b[3], a[0] * b[1] + a[1] * b[0] + a[2] * b[3] - a[3] * b[2],
                     a[0] * b[2] - a[1] * b[3] + a[2] * b[0] + a[3] * b[1], a[0] * b[3] + a[1] * b[2] - a[2] * b[1] + a[3] * b[0]])


def quat2mat(q):
    w, x, y, z = q
    return np.array([[w * w + x * x - y * y - z * z, 2 * (x * y - w * z), 2 * (x * z + w * y)],
                     [2 * (x * y + w * z), w * w - x * x + y * y - z * z, 2 * (y * z - w * x)],
                     [2 * (x * z - w * y), 2 * (y * z + w * x), w * w - x * x - y * y + z * z]])


def measure(sd, row, n, gear, gyro_cut, acc_cut):
    """the measured sensordata [29] from the true one, a sensor row and the tick's 25 draws"""
    out = np.array(sd, dtype=np.float64)
    r = np.asarray(row, dtype=np.float64)
    for c in range(16):
        e = r[SN_ENC_OFF + c] + n[c]
        if c < 10:
            out[DRIVE_S[c]] += gear[c] * e
        else:
            out[JOINT_S[c - 10]] += e
    qm = r[SN_QUAT:SN_QUAT + 4]
    h = np.asarray(n[16:19]) * 0.5
    inv = 1.0 / np.sqrt(1.0 + h[0] * h[0] + h[1] * h[1] + h[2] * h[2])
    dq = np.array([inv, h[0] * inv, h[1] * inv, h[2] * inv])
    out[16:20] = _qmul(_qmul(out[16:20], qm), dq)
    R = quat2mat(qm)
    g = R.T @ out[20:23] + r[SN_GYRO_BIAS:SN_GYRO_BIAS + 3] + np.asarray(n[19:22])
    a = R.T @ out[23:26] + r[SN_ACC_BIAS:SN_ACC_BIAS + 3] + np.asarray(n[22:25])
    out[20:23] = np.clip(g, -gyro_cut, gyro_cut) if gyro_cut > 0 else g
    out[23:26] = np.clip(a, -acc_cut, acc_cut) if acc_cut > 0 else a
    out[26:29] = R.T @ out[26:29]
    return out


class OracleSensors:
    """the sensor model in front of an OracleSim: call step_pd(u, y) instead of the oracle's; the counter advances by one per tick"""

    def __init__(self, o, model, row, key, counter=0):
        t = table(model)
        self.o, self.row, self.key, self.counter = o, np.asarray(row, dtype=np.float64), int(key), int(counter)
        self.gear = t['actuator_gear'][:10]
        self.gyro_cut, self.acc_cut = float(t['sensor_cutoff'][17]), float(t['sensor_cutoff'][18])
        self.std = channel_std(self.row)

    def measure_now(self):
        sd = self.o.arr('sensordata')
        return measure(sd.copy(), self.row, draws(self.key, self.counter, self.std), self.gear, self.gyro_cut, self.acc_cut)

    def step_pd(self, u, y=None):
        self.o.arr('sensordata')[:] = self.measure_now()
        self.o.step_pd(u, y)
        self.counter += 1


# ------------------------------------------------------------------ the host emulation of the F_SN sources (tests/emu/emu_sensors.cpp)
CHAIN_PARENT, CHAIN, PLAIN, PLAIN_PARENT = 1, 2, 3, 4   # emu_sn_mode
_LIB = None


def lib():
    global _LIB
    if _LIB is None:
        import emu_harness as E
        out = os.path.join(E.HERE, 'emu', '_build', 'libcassie_emu_sensors.so')
        srcs = [os.path.join(E.HERE, 'emu', f) for f in ('emu_sensors.cpp', 'emu.cpp')] + \
            [os.path.join(E.CSRC, f) for f in ('mjcf.cpp', 'step_core.inl', 'devmodel.h', 'devbuild.h', 'model.h', 'estimator_host.h', 'cassie_tree_gen.inc')]
        if not os.path.exists(out) or any(os.path.getmtime(out) < os.path.getmtime(f) for f in srcs):
            os.makedirs(os.path.dirname(out), exist_ok=True)
            subprocess.check_call(['g++', '-O1', '-std=c++17', '-fPIC', '-shared', '-o', out + '.tmp', srcs[0], os.path.join(E.CSRC, 'mjcf.cpp')])
            os.replace(out + '.tmp', out)
        L = C.CDLL(out)
        vp, dp, ci, up, ull = C.c_void_p, C.POINTER(C.c_double), C.c_int, C.POINTER(C.c_ulonglong), C.c_ulonglong
        L.emu_sn_new.restype = vp
        L.emu_sn_new.argtypes = [C.c_char_p, ci]
        L.emu_sn_free.argtypes = [vp]
        L.emu_sn_mode.argtypes = [vp, ci]
        L.emu_sn_set_row.argtypes = [vp, dp, ull, ull]
        L.emu_sn_counter.argtypes = [vp]
        L.emu_sn_counter.restype = ull
        L.emu_sn_step.argtypes = [vp, dp, ci]
        L.emu_sn_forward.argtypes = [vp]
        L.emu_sn_philox.argtypes = [up, up, up, up, ci]
        L.emu_sn_noise.argtypes = [dp, up, C.POINTER(C.c_float), dp, ci]
        L.emu_get.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_set.argtypes = [vp, C.c_char_p, dp, ci]
        L.emu_enable_est.argtypes = [vp, ci]
        _LIB = L
    return _LIB


def _dp(a):
    return np.ascontiguousarray(a, dtype=np.float64).ctypes.data_as(C.POINTER(C.c_double))


def emu_philox(t, j, key):
    L = lib()
    t, j, key = [np.ascontiguousarray(v, dtype=np.uint64) for v in (t, j, key)]
    out = np.zeros((len(t), 4), dtype=np.uint64)
    up = C.POINTER(C.c_ulonglong)
    L.emu_sn_philox(t.ctypes.data_as(up), j.ctypes.data_as(up), key.ctypes.data_as(up), out.ctypes.data_as(up), len(t))
    return out


def emu_noise(sigma, word):
    L = lib()
    s, w = np.ascontiguousarray(sigma, dtype=np.float64), np.ascontiguousarray(word, dtype=np.uint64)
    o32, o64 = np.zeros(len(s), dtype=np.float32), np.zeros(len(s))
    L.emu_sn_noise(_dp(s), w.ctypes.data_as(C.POINTER(C.c_ulonglong)), o32.ctypes.data_as(C.POINTER(C.c_float)), o64.ctypes.data_as(C.POINTER(C.c_double)), len(s))
    return o32, o64


class SnSim:
    """one emulated environment running the source of `mode` (emu_sn_mode)"""

    def __init__(self, model_path, mode=CHAIN, fp32=False):
        self.L = lib()
        self.h = self.L.emu_sn_new(model_path.encode(), 1 if fp32 else 0)
        assert self.h
        self.L.emu_sn_mode(self.h, mode)

    def close(self):
        if self.h:
            self.L.emu_sn_free(self.h)
            self.h = None

    def get(self, name, n=4096):
        buf = np.zeros(n)
        k = self.L.emu_get(self.h, name.encode(), buf.ctypes.data_as(C.POINTER(C.c_double)), n)
        assert k >= 0, name
        return buf[:k]

    def set_row(self, row, key=0, counter=0):
        self.L.emu_sn_set_row(self.h, _dp(row), int(key), int(counter))

    def counter(self):
        return int(self.L.emu_sn_counter(self.h))

    def enable_est(self, on=True):
        self.L.emu_enable_est(self.h, 1 if on else 0)

    def step(self, pd50, nticks=1):
        self.L.emu_sn_step(self.h, _dp(pd50), nticks)
