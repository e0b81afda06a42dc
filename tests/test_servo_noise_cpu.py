# SPDX-License-Identifier: Apache-2.0
"""Servo measurement noise (upkie_b200_set_servo_noise): the C struct against its mirror; the sigma draw law, the
cycle counters and the per-cycle normals compiled for the CPU (tests/hostsim/servo_noise.cpp) against a NumPy
statement of include/upkie_b200.h; the statistics of the standardised noise; the view of zero sigmas; the gyropod and
pendulum odometry and reset leg targets of the noisy replies; the spec's validation on both sides and the family the
host picks. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import servo_noise_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
SEED = 0x5E12C0
LEGS = [0, 1, 3, 4]  # hip and knee joints, the order of UPKIE_ST_LEG_TARGET
TAG, CYCLE, RESET = 1 << 55, (1 << 55) | (1 << 54), (1 << 55) | (1 << 54) | (1 << 53)

_LIB = None
fp, u32p, u8p, ip = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.POINTER(C.c_int)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "servo_noise.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_noise_"), "libhostsim_servo_noise.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp, u64 = C.c_void_p, C.c_uint64
        spec_p = C.POINTER(_abi.UpkieServoNoise)
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_servo_noise_draw.argtypes = [spec_p, u64, u64, C.c_uint32, fp]
        L.hostsim_servo_noise_reset.argtypes = [C.c_int, spec_p, u64, u64, u32p, fp, u8p]
        for name in ("hostsim_servo_noise_cycle", "hostsim_servo_noise_reset_cycle", "hostsim_servo_noise_cycle_before"):
            getattr(L, name).restype = u64
        L.hostsim_servo_noise_cycle.argtypes = [C.c_uint32, C.c_uint32]
        L.hostsim_servo_noise_reset_cycle.argtypes = [C.c_uint32]
        L.hostsim_servo_noise_cycle_before.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
        L.hostsim_servo_noise_normals.argtypes = [u64, u64, u64, fp]
        L.hostsim_servo_noise_view.argtypes = [C.c_int, fp, fp, u64, u64, u64, ip]
        L.hostsim_servo_noise_gyropod_obs.argtypes = [vp, C.c_int, fp, fp, u64, u64, u64, fp]
        L.hostsim_servo_noise_spec_error.argtypes = [spec_p] + [C.c_int] * 5 + [C.c_char_p, C.c_int]
        L.hostsim_step_family_servo_noise.argtypes = [C.c_int] * 6 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def make_spec(plo, phi, vlo, vhi):
    s = _abi.UpkieServoNoise()
    s.position_low[:], s.position_high[:] = list(np.broadcast_to(plo, 6)), list(np.broadcast_to(phi, 6))
    s.velocity_low[:], s.velocity_high[:] = list(np.broadcast_to(vlo, 6)), list(np.broadcast_to(vhi, 6))
    return s


def sigma_np(spec, seed, g, k):
    """[len(g), 12] the sigmas of draw k of the envs of global index g (include/upkie_b200.h)"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    kk = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4)
    lo = np.array(list(spec.position_low) + list(spec.velocity_low), dtype=np.float32)
    hi = np.array(list(spec.position_high) + list(spec.velocity_high), dtype=np.float32)
    out = np.zeros(g.shape + (12,), dtype=np.float32)
    for b in range(3):
        w = philox_np(g, np.uint64(TAG) | kk | np.uint64(b), np.full(g.shape, seed, dtype=np.uint64))
        for r in range(4):
            c = 4 * b + r
            out[:, c] = np.minimum(lo[c] + (hi[c] - lo[c]) * u01(w[r]), hi[c])
    return out


def words_np(seed, g, cycle):
    """the twelve Philox words of a cycle: [3 blocks][4]"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    return np.stack([np.stack(philox_np(g, np.uint64(cycle) | np.uint64(b), np.full(g.shape, seed, dtype=np.uint64)))
                     for b in range(3)])


def normals_np(seed, g, cycle):
    """[len(g), 12] the normals of a cycle: gaussian8's Box-Muller transform, in float32"""
    w = words_np(seed, g, cycle)
    out = np.zeros((w.shape[2], 12), dtype=np.float32)
    for b in range(3):
        for p in range(2):
            u1 = ((w[b, 2 * p] >> np.uint32(8)).astype(np.float32) + np.float32(1)) * np.float32(1.0 / 16777216.0)
            u2 = u01(w[b, 2 * p + 1])
            rad = np.sqrt(np.float32(-2) * np.log(u1))
            ang = np.float32(6.28318530718) * u2
            out[:, 4 * b + 2 * p] = rad * np.cos(ang)
            out[:, 4 * b + 2 * p + 1] = rad * np.sin(ang)
    return out


def normals_c(seed, g, cycle):
    n = np.zeros(12, dtype=np.float32)
    _lib().hostsim_servo_noise_normals(seed, g, cycle, _p(n))
    return n


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieServoNoise \{(.*?)\} UpkieServoNoise;", header, re.S).group(1)
    names = re.findall(r"\b(\w+)\[6\]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _abi.UpkieServoNoise._fields_]
    assert C.sizeof(_abi.UpkieServoNoise) == 96


def test_sigma_draws_match_the_numpy_law():
    spec = make_spec([0.0, 0.01, 0.0, 0.002, 0.0, 0.05], [0.01, 0.02, 0.0, 0.004, 0.1, 0.05],
                     [0.1, 0.0, 0.5, 0.0, 0.0, 1.0], [0.2, 0.0, 1.0, 5.0, 0.3, 2.0])
    g = np.arange(3, 67, dtype=np.uint64)
    s = np.zeros(12, dtype=np.float32)
    for k in (1, 2, 999, 2 ** 31 + 5):
        ref = sigma_np(spec, SEED, g, k)
        got = np.zeros((len(g), 12), dtype=np.float32)
        for i, x in enumerate(g):
            _lib().hostsim_servo_noise_draw(C.byref(spec), SEED, int(x), k, _p(s))
            got[i] = s
        np.testing.assert_array_equal(got, ref)
        lo = np.array(list(spec.position_low) + list(spec.velocity_low), np.float32)
        hi = np.array(list(spec.position_high) + list(spec.velocity_high), np.float32)
        assert (got >= lo).all() and (got <= hi).all()
        assert (got[:, 2] == 0).all() and (got[:, 7] == 0).all()  # zero ranges: exactly 0
    # the ranges of one column change no other column's draw
    b = sigma_np(make_spec(0.0, 0.1, 0.0, 5.0), SEED, g, 7)
    spec2 = make_spec(0.0, 0.1, 0.0, 5.0)
    spec2.position_high[3] = 0.0
    c = sigma_np(spec2, SEED, g, 7)
    keep = [j for j in range(12) if j != 3]
    np.testing.assert_array_equal(c[:, keep], b[:, keep])
    assert (c[:, 3] == 0).all()


def test_reset_counts_stores_and_marks():
    n = 40
    spec = make_spec(0.0, 0.01, 0.0, 0.5)
    count = np.full(n, 6, dtype=np.uint32)
    sigma = np.zeros((12, n), dtype=np.float32)
    fresh = np.zeros(n, dtype=np.uint8)
    _lib().hostsim_servo_noise_reset(n, C.byref(spec), SEED, 200, _p(count, u32p), _p(sigma), _p(fresh, u8p))
    assert (count == 7).all() and (fresh == 1).all()
    np.testing.assert_array_equal(sigma.T, sigma_np(spec, SEED, 200 + np.arange(n), 7))


def test_cycle_counters():
    L = _lib()
    assert L.hostsim_servo_noise_cycle(0, 0) == CYCLE
    assert L.hostsim_servo_noise_cycle(17, 3) == CYCLE | (17 << 20) | (3 << 2)
    assert L.hostsim_servo_noise_cycle(2 ** 32 - 1, 4) == CYCLE | ((2 ** 32 - 1) << 20) | (4 << 2)
    assert L.hostsim_servo_noise_reset_cycle(9) == RESET | (9 << 2)
    # a reset cycle never coincides with a step cycle: bit 53 is above every step cycle's bits
    assert (L.hostsim_servo_noise_cycle(2 ** 32 - 1, 2 ** 18 - 1) | 3) < RESET
    # the cycle `age` substeps before cycle nb - 1 of tick t
    nb = 5
    for t in (3, 10, 1000):
        for age in range(0, 23):
            c = t * nb + nb - 1 - age
            assert L.hostsim_servo_noise_cycle_before(t, nb, age) == L.hostsim_servo_noise_cycle(c // nb, c % nb)
    # before tick 0: the tick counter wraps
    assert L.hostsim_servo_noise_cycle_before(0, nb, nb) == L.hostsim_servo_noise_cycle(2 ** 32 - 1, nb - 1)


def test_normals_match_the_restatement():
    g = np.arange(0, 8, dtype=np.uint64)
    for cycle in (CYCLE | (5 << 20) | (2 << 2), CYCLE | (123456 << 20), RESET | (4 << 2)):
        ref = normals_np(SEED, g, cycle)
        for i, x in enumerate(g):
            got = normals_c(SEED, int(x), cycle)
            # the uniforms are bit for bit the restatement's; log / sincos round within an ulp or two of NumPy's
            np.testing.assert_allclose(got, ref[i], rtol=2e-6, atol=2e-6)
            assert np.isfinite(got).all()
    # the reset cycle of draw k and step cycles draw different normals
    a = normals_c(SEED, 3, RESET | (1 << 2))
    for t in range(4):
        for s in range(5):
            assert not np.array_equal(a, normals_c(SEED, 3, CYCLE | (t << 20) | (s << 2)))


def test_normals_statistics():
    n = 20000
    rows = np.stack([normals_c(SEED, g, CYCLE | (t << 20) | (s << 2))
                     for g in range(4) for t in range(n // 20) for s in range(5)])
    assert rows.shape == (n, 12)
    m, sd = rows.mean(axis=0), rows.std(axis=0)
    assert np.abs(m).max() < 0.04, m
    assert np.abs(sd - 1).max() < 0.03, sd
    corr = np.corrcoef(rows.T)
    off = corr[~np.eye(12, dtype=bool)]
    assert np.abs(off).max() < 0.04, np.abs(off).max()
    # tails of a normal
    assert 0.0022 < (np.abs(rows) > 3).mean() < 0.0032  # 0.0027 for a standard normal


def test_view_adds_sigma_times_the_normal_and_zero_sigma_leaves_every_bit():
    rng = np.random.default_rng(21)
    n = 32
    state = rng.normal(0.0, 0.5, (n, _abi.STATE_DIM)).astype(np.float32)
    state[:8, _abi.ST_Q:_abi.ST_Q + 6] = -0.0  # a sum with +0 would turn -0 into +0
    state[:8, _abi.ST_QD:_abi.ST_QD + 6] = -0.0
    view = state.copy()
    changed = np.zeros(n, dtype=np.int32)
    cyc = CYCLE | (11 << 20) | (4 << 2)
    _lib().hostsim_servo_noise_view(n, _p(view), _p(np.zeros((n, 12), np.float32)), SEED, 0, cyc, _p(changed, ip))
    assert view.tobytes() == state.tobytes() and not changed.any()
    sigma = rng.uniform(0.0, 0.01, (n, 12)).astype(np.float32)
    sigma[:, 6:] *= 50
    sigma[:, [2, 5, 8, 11]] = 0.0  # no wheel noise: the odometry is unchanged
    _lib().hostsim_servo_noise_view(n, _p(view), _p(sigma), SEED, 0, cyc, _p(changed, ip))
    assert not changed.any()
    for i in range(n):
        nn = normals_c(SEED, i, cyc)
        inc = sigma[i] * nn
        q, qd = state[i, _abi.ST_Q:_abi.ST_Q + 6], state[i, _abi.ST_QD:_abi.ST_QD + 6]
        np.testing.assert_array_equal(view[i, _abi.ST_Q:_abi.ST_Q + 6], np.where(inc[:6] != 0, q + inc[:6], q))
        np.testing.assert_array_equal(view[i, _abi.ST_QD:_abi.ST_QD + 6], np.where(inc[6:] != 0, qd + inc[6:], qd))
    rest = np.ones(_abi.STATE_DIM, bool)
    rest[_abi.ST_Q:_abi.ST_Q + 6] = rest[_abi.ST_QD:_abi.ST_QD + 6] = False
    assert view[:, rest].tobytes() == state[:, rest].tobytes()
    sigma[:, 11] = 0.3
    _lib().hostsim_servo_noise_view(n, _p(state.copy()), _p(sigma), SEED, 0, cyc, _p(changed, ip))
    assert changed.all()


class _Sim:
    def __init__(self):
        self._m = default_model().to_struct()
        self._c = _abi.default_sim_config()
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h

    def __del__(self):
        try:
            _lib().hostsim_destroy(self.h)
        except Exception:
            pass


def test_gyropod_odometry_and_leg_targets_are_the_noisy_replies():
    rng = np.random.default_rng(22)
    n = 16
    sim = _Sim()
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    state[:, 3] = 1.0
    state[:, _abi.ST_Q:_abi.ST_Q + 6] = rng.uniform(-0.3, 0.3, (n, 6))
    state[:, _abi.ST_QD:_abi.ST_QD + 6] = rng.uniform(-2.0, 2.0, (n, 6))
    sigma = np.concatenate([rng.uniform(0, 0.01, (n, 6)), rng.uniform(0, 0.5, (n, 6))], axis=1).astype(np.float32)
    cyc = RESET | (3 << 2)
    plain = state.copy()
    obs, plain_obs = np.zeros((n, 6), np.float32), np.zeros((n, 6), np.float32)
    _lib().hostsim_servo_noise_gyropod_obs(sim.h, n, _p(state), _p(sigma), SEED, 0, cyc, _p(obs))
    _lib().hostsim_servo_noise_gyropod_obs(sim.h, n, _p(plain), _p(np.zeros_like(sigma)), SEED, 0, cyc, _p(plain_obs))
    model = default_model()
    sr = np.float32((1.0 if model.left_wheeled else -1.0) * model.wheel_radius)
    noisy_q = np.zeros((n, 6), np.float32)
    noisy_qd = np.zeros((n, 6), np.float32)
    for i in range(n):
        inc = sigma[i] * normals_c(SEED, i, cyc)
        noisy_q[i] = state[i, _abi.ST_Q:_abi.ST_Q + 6] + inc[:6]
        noisy_qd[i] = state[i, _abi.ST_QD:_abi.ST_QD + 6] + inc[6:]
    np.testing.assert_array_equal(obs[:, 0], np.float32(0.5) * (noisy_q[:, 2] - noisy_q[:, 5]) * sr)
    np.testing.assert_array_equal(obs[:, 3], np.float32(0.5) * (noisy_qd[:, 2] - noisy_qd[:, 5]) * sr)
    np.testing.assert_array_equal(obs[:, [1, 2, 4, 5]], plain_obs[:, [1, 2, 4, 5]])  # pitch, yaw and rates
    # the leg targets a reset sets are the reported hip and knee positions of the reset observation
    lt = slice(_abi.ST_LEG_TARGET, _abi.ST_LEG_TARGET + 4)
    np.testing.assert_array_equal(state[:, lt], noisy_q[:, LEGS])
    np.testing.assert_array_equal(plain[:, lt], plain[:, _abi.ST_Q + np.array(LEGS)])


def _why(spec, limits=1, spine=0, body=0, delay=0, drop=0):
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_servo_noise_spec_error(C.byref(spec), limits, spine, body, delay, drop, buf, 256)
    return buf.value.decode() if r else None


def test_spec_rejections():
    ok = make_spec(0.0, 0.01, 0.0, 0.5)
    assert _why(ok) is None
    assert _why(make_spec(0.1, 0.1, 5.0, 5.0)) is None
    assert _why(make_spec(0.0, 0.0, 0.0, 0.0)) is None
    assert _why(ok, delay=1) is None and _why(ok, drop=1) is None
    bad = ("set_servo_noise: every range must be finite with 0 <= low <= high, position high <= 0.1 rad and velocity "
           "high <= 5 rad/s")
    nan, inf = float("nan"), float("inf")
    for args in ((nan, 0.01, 0.0, 0.5), (0.0, inf, 0.0, 0.5), (0.0, 0.01, -inf, 0.5), (0.0, 0.01, 0.0, nan),
                 (-0.001, 0.01, 0.0, 0.5), (0.0, 0.01, -0.1, 0.5), (0.02, 0.01, 0.0, 0.5), (0.0, 0.01, 0.6, 0.5),
                 (0.0, 0.11, 0.0, 0.5), (0.0, 0.01, 0.0, 5.01)):
        assert _why(make_spec(*args)) == bad, args
    one = make_spec(0.0, 0.01, 0.0, 0.5)
    one.velocity_high[4] = 6.0
    assert _why(one) == bad
    assert _why(ok, limits=0) == ("set_servo_noise: needs joint_limits != 0 (the noise runs in the observation-delay "
                                  "kernels)")
    assert _why(ok, spine=1) == "set_servo_noise: spine_mode reports the spine's own servos"
    assert _why(ok, body=1) == "set_servo_noise: body_contacts has no servo-noise kernels"
    assert _why(ok, delay=1, drop=1) == ("set_servo_noise: not with both an observation delay and servo dropouts (a "
                                         "delayed snapshot does not record which of its replies were held)")


def _family(limits=1, spine=0, body=0, obs_delay=0, mode=0, transport=0):
    buf = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_servo_noise(limits, spine, body, obs_delay, mode, transport, buf, 256)
    return f, buf.value.decode()


def test_family_choice():
    for mode in range(3):
        for transport in (0, 1):
            assert _family(mode=mode, transport=transport)[0] == FAM_SENSE
            assert _family(mode=mode, transport=transport, obs_delay=1)[0] == FAM_SENSE
    assert _family(transport=2) == (
        -1, "servo noise has no in-kernel rollout transport (use upkie_b200_step with compact rows)")
    assert _family(spine=1) == (-1, "servo noise: spine_mode reports the spine's own servos")
    assert _family(limits=0) == (-1, "servo noise needs joint_limits != 0")
    assert _family(body=1) == (-1, "servo noise has no body-contact kernels")


def test_python_spec_parsing():
    s = servo_noise_spec({"position": 0.002, "velocity": (0.0, 0.5)})
    assert list(s.position_low) == [np.float32(0.002)] * 6 and list(s.position_high) == [np.float32(0.002)] * 6
    assert list(s.velocity_low) == [0.0] * 6 and list(s.velocity_high) == [np.float32(0.5)] * 6
    s = servo_noise_spec({"velocity": {"left_wheel": 0.3, "right_wheel": (0.1, 0.2)}})
    assert list(s.position_high) == [0.0] * 6
    assert list(s.velocity_low) == [0, 0, np.float32(0.3), 0, 0, np.float32(0.1)]
    assert list(s.velocity_high) == [0, 0, np.float32(0.3), 0, 0, np.float32(0.2)]
    assert servo_noise_spec(None) is None
    assert servo_noise_spec({"position": 0.1, "velocity": 5.0}) is not None
    for bad in ({"position": (0.02, 0.01)}, {"position": 0.2}, {"velocity": 5.5}, {"velocity": -0.1},
                {"position": float("nan")}, {"velocity": (0.0, float("inf"))}, {"position": "x"},
                {"position": (0.1, 0.2, 0.3)}, {"position": ("a", 0.1)}, 0.01, (0.0, 0.1)):
        with pytest.raises(UpkieException, match="servo_noise"):
            servo_noise_spec(bad)
    with pytest.raises(UpkieException, match="servo_noise: unknown key"):
        servo_noise_spec({"torque": 0.1})
    with pytest.raises(UpkieException, match="servo_noise: velocity: unknown joint"):
        servo_noise_spec({"velocity": {"left_elbow": 0.1}})
    for kw, what in (({"spine_mode": True}, "spine_mode"), ({"joint_limits": 0}, "joint_limits"),
                     ({"body_contacts": True}, "body_contacts"),
                     ({"observation_delay": True, "servo_dropout": True}, "observation delay")):
        with pytest.raises(UpkieException, match=f"servo_noise: .*{what}"):
            servo_noise_spec({"position": 0.01}, **kw)
    assert servo_noise_spec({"position": 0.01}, observation_delay=True) is not None
