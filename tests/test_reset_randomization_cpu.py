# SPDX-License-Identifier: Apache-2.0
"""Reset randomisation (upkie_b200_set_reset_randomization): the C struct against its mirror, the B200VectorEnv dict
forms, and the draw the kernels run, compiled for the CPU (tests/hostsim/reset_randomization.cpp), against a NumPy
statement of the draw law. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import reset_randomization_spec

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")


def test_constants_and_struct_match_the_header():
    header = open(HEADER).read()
    defs = dict(re.findall(r"#define (UPKIE_\w+) (\d+)", header))
    assert int(defs["UPKIE_RR_INERTIA"]) == _abi.RR_INERTIA == _abi.EP_DIM
    assert int(defs["UPKIE_RR_FRICTION"]) == _abi.RR_FRICTION == _abi.RR_INERTIA + 6
    assert int(defs["UPKIE_RR_DIM"]) == _abi.RR_DIM == _abi.RR_FRICTION + 1
    body = re.search(r"typedef struct UpkieResetRandomization \{(.*?)\} UpkieResetRandomization;", header, re.S).group(1)
    assert re.findall(r"(\w+)(?:\[\w+\])?;", body) == [f for f, _ in _abi.UpkieResetRandomization._fields_]
    S = _abi.UpkieResetRandomization
    assert (S.columns.offset, S.low.offset, S.high.offset, C.sizeof(S)) == (0, 8, 8 + 4 * 35, 8 + 8 * 35)


# ---- dict -> spec ---------------------------------------------------------------------------------------------------


def _selected(spec):
    return [k for k in range(_abi.RR_DIM) if (spec.columns >> k) & 1]


def test_every_argument_form():
    s = reset_randomization_spec({
        "inertia_variation": 0.2,
        "floor_friction": (0.5, 1.2),
        "torque_control_kp": (15.0, 25.0),
        "torque_control_kd": (0.5, 1.5),
        "joint_properties": {"left_knee": {"friction": (0.0, 0.05), "torque_control_noise": (0.0, 0.1)},
                             "right_wheel": {"torque_measurement_noise": (0.01, 0.02)}},
        "imu_uncertainty": {"accelerometer_bias": ((-0.1, -0.2, -0.3), (0.1, 0.2, 0.3)), "accelerometer_noise": (0, 0.05),
                            "gyroscope_bias": (-0.01, 0.01), "gyroscope_noise": (0.0, 0.002)},
    })
    J = _abi.JOINT_NAMES
    expect = {
        _abi.EP_KP: (15.0, 25.0), _abi.EP_KD: (0.5, 1.5),
        _abi.EP_FRICTION + J.index("left_knee"): (0.0, 0.05), _abi.EP_CTRL_NOISE + J.index("left_knee"): (0.0, 0.1),
        _abi.EP_MEAS_NOISE + J.index("right_wheel"): (0.01, 0.02),
        _abi.EP_IMU_ACC_BIAS: (-0.1, 0.1), _abi.EP_IMU_ACC_BIAS + 1: (-0.2, 0.2), _abi.EP_IMU_ACC_BIAS + 2: (-0.3, 0.3),
        _abi.EP_IMU_ACC_NOISE: (0.0, 0.05), _abi.EP_IMU_GYRO_NOISE: (0.0, 0.002),
        _abi.RR_FRICTION: (0.5, 1.2),
    }
    expect.update({_abi.EP_IMU_GYRO_BIAS + k: (-0.01, 0.01) for k in range(3)})
    expect.update({_abi.RR_INERTIA + b: (-0.2, 0.2) for b in range(6)})
    assert _selected(s) == sorted(expect)
    for k, (lo, hi) in expect.items():
        assert (s.low[k], s.high[k]) == (np.float32(lo), np.float32(hi)), k
    assert reset_randomization_spec(None) is None
    assert _selected(reset_randomization_spec({})) == []


@pytest.mark.parametrize("spec", [
    {"inertia": 0.1},                                                  # unknown key
    {"joint_properties": {"left_ankle": {"friction": (0, 1)}}},        # unknown joint
    {"joint_properties": {"left_hip": {"damping": (0, 1)}}},           # unknown field
    {"imu_uncertainty": {"magnetometer_bias": (0, 1)}},                # unknown IMU key
    {"torque_control_kp": (25.0, 15.0)},                               # low > high
    {"torque_control_kd": (-0.1, 1.0)},                                # negative gain
    {"joint_properties": {"left_hip": {"torque_control_noise": (-0.1, 0.1)}}},
    {"floor_friction": (-0.1, 1.0)},
    {"floor_friction": (0.5, np.inf)},
    {"torque_control_kp": (np.nan, 1.0)},
    {"inertia_variation": 1.0},                                        # bound <= -1
    {"inertia_variation": -0.1},
    {"imu_uncertainty": {"gyroscope_noise": (-1e-3, 0.0)}},
    {"imu_uncertainty": {"accelerometer_bias": ((0, 0), (1, 1))}},     # not one or three axes
    {"torque_control_kp": 20.0},                                       # not a pair
])
def test_bad_specs_are_rejected_before_the_device(spec):
    from upkie_b200.envs import B200VectorEnv

    with pytest.raises((UpkieException, ValueError)):
        reset_randomization_spec(spec)
    with pytest.raises((UpkieException, ValueError)):
        B200VectorEnv(4, "servos", reset_randomization=spec)  # no device here: rejected before it is needed


# ---- the draw on the CPU build of the kernels' code --------------------------------------------------------------------

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "reset_randomization.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_rr_"), "libhostsim_rr.so")
        # tools/hostsim_sanitizers.sh sets the flags of an AddressSanitizer / UBSan build
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        sp, fp = C.POINTER(_abi.UpkieResetRandomization), C.POINTER(C.c_float)
        u32p, u8p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)
        L.hostsim_rr_draw.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_uint32, fp]
        L.hostsim_rr_reset.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_int, u8p, u32p, fp, fp, fp]
        L.hostsim_rr_flags.argtypes = [sp]
        L.hostsim_rr_flags.restype = C.c_uint32
        L.hostsim_philox.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, u32p]
        _LIB = L
    return _LIB


def philox_np(counter_lo, counter_hi, key):
    """Philox4x32-10 (Salmon et al., SC'11) on arrays of 64-bit counter words and keys"""
    lo, hi, key = (np.asarray(x, dtype=np.uint64) for x in (counter_lo, counter_hi, key))
    m32 = np.uint64(0xFFFFFFFF)
    c = [lo & m32, lo >> np.uint64(32), hi & m32, hi >> np.uint64(32)]
    k0, k1 = key & m32, key >> np.uint64(32)
    for _ in range(10):
        p0, p1 = np.uint64(0xD2511F53) * c[0], np.uint64(0xCD9E8D57) * c[2]
        c = [(p1 >> np.uint64(32)) ^ c[1] ^ k0, p1 & m32, (p0 >> np.uint64(32)) ^ c[3] ^ k1, p0 & m32]
        k0, k1 = (k0 + np.uint64(0x9E3779B9)) & m32, (k1 + np.uint64(0xBB67AE85)) & m32
    return [x.astype(np.uint32) for x in c]


def draw_np(spec, seed, env_index, draw):
    """The draw law of include/upkie_b200.h in NumPy fp32: values [len(env_index), RR_DIM]"""
    env_index = np.atleast_1d(np.asarray(env_index, dtype=np.uint64))
    draw = np.broadcast_to(np.asarray(draw, dtype=np.uint64), env_index.shape)
    low = np.ctypeslib.as_array(spec.low).astype(np.float32)
    high = np.ctypeslib.as_array(spec.high).astype(np.float32)
    out = np.empty((env_index.size, _abi.RR_DIM), dtype=np.float32)
    for b in range(9):
        hi_word = np.uint64(1 << 63) | (draw << np.uint64(4)) | np.uint64(b)
        words = philox_np(env_index, hi_word, np.full(env_index.shape, seed, dtype=np.uint64))
        for k in range(4):
            c = 4 * b + k
            if c >= _abi.RR_DIM:
                break
            u = (words[k] >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
            out[:, c] = np.minimum(low[c] + (high[c] - low[c]) * u, high[c])
    return out


def _spec(seed=0, columns=(1 << _abi.RR_DIM) - 1):
    rng = np.random.default_rng(seed)
    s = _abi.UpkieResetRandomization()
    s.columns = columns
    lo = rng.uniform(0.0, 2.0, _abi.RR_DIM)
    hi = lo + rng.uniform(0.0, 3.0, _abi.RR_DIM)
    lo[_abi.EP_IMU_ACC_BIAS:_abi.EP_IMU_ACC_BIAS + 3] -= 2.0  # biases may be negative
    lo[_abi.RR_INERTIA:_abi.RR_FRICTION], hi[_abi.RR_INERTIA:_abi.RR_FRICTION] = -0.3, 0.3
    hi[5] = lo[5]  # an empty range
    for k in range(_abi.RR_DIM):
        s.low[k], s.high[k] = lo[k], hi[k]
    return s


def test_numpy_philox_matches_the_kernels():
    L = _lib()
    rng = np.random.default_rng(1)
    for _ in range(20):
        lo, hi, key = (int(x) for x in rng.integers(0, 2**63, 3, dtype=np.uint64))
        out = (C.c_uint32 * 4)()
        L.hostsim_philox(lo, hi | (1 << 63), key, out)
        assert [int(w[0]) for w in philox_np([lo], [hi | (1 << 63)], [key])] == list(out)


@pytest.mark.parametrize("seed", [0, 7, 2**40 + 3])
def test_draw_matches_the_numpy_law(seed):
    L = _lib()
    spec = _spec(seed)
    for env in (0, 1, 4095, 65535, 2**33 + 17):
        for d in (1, 2, 3, 1000, 2**32 - 1):
            v = np.empty(_abi.RR_DIM, dtype=np.float32)
            L.hostsim_rr_draw(C.byref(spec), seed, env, d, v.ctypes.data_as(C.POINTER(C.c_float)))
            np.testing.assert_array_equal(v, draw_np(spec, seed, env, d)[0])
            low, high = np.ctypeslib.as_array(spec.low), np.ctypeslib.as_array(spec.high)
            assert np.all(v >= low) and np.all(v <= high)
    # different draws, envs and seeds give different values
    a, b = draw_np(spec, seed, [3, 3, 4], [1, 2, 1]), draw_np(spec, seed + 1, [3], [1])
    assert not np.array_equal(a[0], a[1]) and not np.array_equal(a[0], a[2]) and not np.array_equal(a[0], b[0])


def _reset(spec, seed, env_offset, n, mask, draws, table, eps, mu):
    fp = C.POINTER(C.c_float)
    _lib().hostsim_rr_reset(C.byref(spec), seed, env_offset, n,
                            mask.ctypes.data_as(C.POINTER(C.c_uint8)) if mask is not None else None,
                            draws.ctypes.data_as(C.POINTER(C.c_uint32)), table.ctypes.data_as(fp), eps.ctypes.data_as(fp),
                            mu.ctypes.data_as(fp))


def test_reset_writes_the_selected_columns_only():
    n, seed, off = 7, 11, 100
    rng = np.random.default_rng(2)
    cols = [_abi.EP_KD, _abi.EP_MEAS_NOISE + 3, _abi.EP_IMU_GYRO_BIAS + 1, _abi.RR_INERTIA + 2, _abi.RR_FRICTION]
    spec = _spec(3, sum(1 << c for c in cols))
    table = rng.uniform(0, 1, (_abi.EP_DIM, n)).astype(np.float32)
    eps = rng.uniform(-0.1, 0.1, (n, 6)).astype(np.float32)
    mu = rng.uniform(0.5, 1.0, n).astype(np.float32)
    draws = np.array([0, 5, 0, 1, 2, 0, 9], dtype=np.uint32)
    mask = np.array([1, 1, 0, 1, 0, 1, 1], dtype=np.uint8)
    t0, e0, m0, d0 = table.copy(), eps.copy(), mu.copy(), draws.copy()
    _reset(spec, seed, off, n, mask, draws, table, eps, mu)
    sel = mask.astype(bool)
    np.testing.assert_array_equal(draws, np.where(sel, d0 + 1, d0))
    full = draw_np(spec, seed, off + np.arange(n), draws)  # every env's current draw
    for k in range(_abi.EP_DIM):
        expect = np.where(sel, full[:, k], t0[k]) if k in cols else t0[k]
        np.testing.assert_array_equal(table[k], expect, err_msg=str(k))
    for b in range(6):
        c = _abi.RR_INERTIA + b
        np.testing.assert_array_equal(eps[:, b], np.where(sel, full[:, c], e0[:, b]) if c in cols else e0[:, b])
    np.testing.assert_array_equal(mu, np.where(sel, full[:, _abi.RR_FRICTION], m0))
    # selecting another column changes no value of this one
    other = _spec(3, spec.columns | (1 << _abi.EP_KP))
    np.testing.assert_array_equal(draw_np(other, seed, off, 4)[0], draw_np(spec, seed, off, 4)[0])


def test_validation_and_noise_flags():
    L = _lib()
    invalid, ctrl, meas, imu = 1, 2, 4, 8

    def flags(**ranges):
        s = _abi.UpkieResetRandomization()
        for k, (lo, hi) in ranges.items():
            c = int(k[1:])
            s.columns |= 1 << c
            s.low[c], s.high[c] = lo, hi
        return L.hostsim_rr_flags(C.byref(s))

    assert flags() == 0
    assert flags(c0=(10.0, 30.0)) == 0
    assert flags(**{f"c{_abi.EP_CTRL_NOISE}": (0.0, 0.1)}) == ctrl
    assert flags(**{f"c{_abi.EP_MEAS_NOISE + 5}": (0.0, 0.1)}) == meas
    assert flags(**{f"c{_abi.EP_IMU_GYRO_BIAS}": (-0.1, 0.0)}) == imu
    assert flags(**{f"c{_abi.EP_IMU_ACC_NOISE}": (0.0, 0.1)}) == imu
    assert flags(**{f"c{_abi.EP_IMU_ACC_NOISE}": (0.0, 0.0)}) == 0
    for bad in ({"c1": (-0.5, 1.0)}, {"c3": (1.0, 0.5)}, {"c2": (0.0, float("inf"))}, {"c20": (float("nan"), 0.0)},
                {f"c{_abi.RR_INERTIA}": (-1.0, 0.0)}, {f"c{_abi.RR_FRICTION}": (-0.1, 1.0)}):
        assert flags(**bad) & invalid, bad
    s = _abi.UpkieResetRandomization()
    s.columns = 1 << _abi.RR_DIM  # no such column
    assert L.hostsim_rr_flags(C.byref(s)) & invalid
