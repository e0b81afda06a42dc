# SPDX-License-Identifier: Apache-2.0
"""Servo encoder zero offsets (upkie_b200_set_encoder_offset): the C struct against its mirror; the draw law and the
reset compiled for the CPU (tests/hostsim/encoder_offset.cpp) against a NumPy statement of include/upkie_b200.h; one
servo tick with offsets against the same tick without them whose targets are shifted on the host; the gyropod's reset
leg targets and their decay toward the servo zero; the family the host picks with offsets set; the spec's validation on
both sides. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import encoder_offset_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
SEED = 0x0FF5E7
LEGS = [0, 1, 3, 4]  # hip and knee joints, the order of UPKIE_ST_LEG_TARGET
ALL = 0x3F
A_POS, A_VEL, A_KP, A_KD, A_MAXT = (_abi.ACT_KEYS.index(k) for k in (
    "position", "velocity", "kp_scale", "kd_scale", "maximum_torque"))

_LIB = None
fp, u32p, ip = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_int)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "encoder_offset.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_enc_"), "libhostsim_encoder_offset.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        spec_p = C.POINTER(_abi.UpkieEncoderOffset)
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_encoder_offset_draw.argtypes = [spec_p, C.c_uint64, C.c_uint64, C.c_uint32, fp]
        L.hostsim_encoder_offset_reset.argtypes = [C.c_int, spec_p, C.c_uint64, C.c_uint64, u32p, fp]
        L.hostsim_encoder_offset_servo_tick.argtypes = [vp, C.c_int, fp, fp, fp, fp]
        L.hostsim_encoder_offset_gyropod_tick.argtypes = [vp, C.c_int, fp, fp, fp, fp, fp]
        L.hostsim_encoder_offset_reset_robot.argtypes = [vp, C.c_int, fp, fp, fp]
        L.hostsim_encoder_offset_view.argtypes = [C.c_int, fp, fp, ip]
        L.hostsim_encoder_offset_spec_error.argtypes = [spec_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_step_family_encoder_offset.argtypes = [C.c_int] * 6 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def offsets_np(spec, seed, g, k):
    """[len(g), 6] the offsets of draw k of the envs of global index g (include/upkie_b200.h): fp32, the product
    rounded on its own, clamped to high; exactly 0 outside the mask"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    kk = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4)
    lo, hi = np.float32(spec.low), np.float32(spec.high)
    out = np.zeros(g.shape + (6,), dtype=np.float32)
    for b in range(2):
        w = philox_np(g, np.uint64(1 << 56) | kk | np.uint64(b), np.full(g.shape, seed, dtype=np.uint64))
        for r in range(4):
            j = 4 * b + r
            if j < 6 and (spec.joint_mask >> j) & 1:
                out[:, j] = np.minimum(lo + (hi - lo) * u01(w[r]), hi)
    return out


class _Sim:
    def __init__(self):
        self._m = default_model().to_struct()
        self._c = _abi.default_sim_config()
        self.P = self._c
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h

    def __del__(self):
        try:
            _lib().hostsim_destroy(self.h)
        except Exception:
            pass


def _standing(n, rng):
    """post-reset states of n robots standing from slightly perturbed initial poses"""
    sim = _Sim()
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, _abi.INIT_POS + 2] = 0.6
    init[:, _abi.INIT_QUAT] = 1.0
    init[:, _abi.INIT_Q:_abi.INIT_Q + 6] = rng.uniform(-0.2, 0.2, (n, 6))
    _lib().hostsim_encoder_offset_reset_robot(sim.h, n, _p(state), _p(init), None)
    return sim, state, init


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieEncoderOffset \{(.*?)\} UpkieEncoderOffset;", header, re.S).group(1)
    names = re.findall(r"\b(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _abi.UpkieEncoderOffset._fields_]
    assert C.sizeof(_abi.UpkieEncoderOffset) == 16


@pytest.mark.parametrize("mask", [ALL, 0b011011, 0b100100, 0b010000])
def test_draws_match_the_numpy_law(mask):
    spec = _abi.UpkieEncoderOffset(-0.07, 0.03, mask, 0)
    g = np.arange(5, 69, dtype=np.uint64)
    d = np.zeros(6, dtype=np.float32)
    for k in (1, 2, 1000, 2 ** 31 + 3):
        ref = offsets_np(spec, SEED, g, k)
        got = np.zeros((len(g), 6), dtype=np.float32)
        for i, x in enumerate(g):
            _lib().hostsim_encoder_offset_draw(C.byref(spec), SEED, int(x), k, _p(d))
            got[i] = d
        np.testing.assert_array_equal(got, ref)
        inside = [(mask >> j) & 1 == 1 for j in range(6)]
        assert (got[:, inside] >= np.float32(-0.07)).all() and (got[:, inside] <= np.float32(0.03)).all()
        # masked-out joints are exactly +0
        out = got[:, [not x for x in inside]]
        assert (out == 0).all() and not np.signbit(out).any()
        # both counters of a draw: joints 0-3 (j / 4 = 0) and 4-5 (j / 4 = 1) vary across envs
        for j in range(6):
            if inside[j]:
                assert len(np.unique(got[:, j])) == len(g)
    # a mask changes no other joint's draw
    full = offsets_np(_abi.UpkieEncoderOffset(-0.07, 0.03, ALL, 0), SEED, g, 7)
    part = offsets_np(spec, SEED, g, 7)
    keep = [j for j in range(6) if (mask >> j) & 1]
    np.testing.assert_array_equal(part[:, keep], full[:, keep])


def test_degenerate_range_is_that_offset():
    spec = _abi.UpkieEncoderOffset(0.02, 0.02, ALL, 0)
    d = np.zeros(6, dtype=np.float32)
    _lib().hostsim_encoder_offset_draw(C.byref(spec), SEED, 3, 9, _p(d))
    np.testing.assert_array_equal(d, np.float32(0.02))


def test_reset_counts_and_stores_the_draw():
    n = 40
    spec = _abi.UpkieEncoderOffset(-0.05, 0.05, 0b011011, 0)
    count = np.full(n, 4, dtype=np.uint32)
    offset = np.zeros((6, n), dtype=np.float32)
    _lib().hostsim_encoder_offset_reset(n, C.byref(spec), SEED, 100, _p(count, u32p), _p(offset))
    assert (count == 5).all()
    np.testing.assert_array_equal(offset.T, offsets_np(spec, SEED, 100 + np.arange(n), 5))
    # sharding: the draw is keyed on the global env index
    np.testing.assert_array_equal(offset.T[20:], offsets_np(spec, SEED, 120 + np.arange(20), 5))


def test_servo_tick_is_the_shifted_twin():
    rng = np.random.default_rng(11)
    n = 64
    sim, state, _ = _standing(n, rng)
    twin_state = state.copy()
    lo, hi = np.array(default_model().q_lower, np.float32), np.array(default_model().q_upper, np.float32)
    action = np.zeros((n, 6, 6), dtype=np.float32)
    action[:, :, A_POS] = rng.uniform(np.maximum(lo, -2.0) + 0.15, np.minimum(hi, 2.0) - 0.15, (n, 6))
    action[:, [2, 5], A_POS] = np.nan  # the wheels: velocity control
    action[:, :, A_VEL] = rng.uniform(-1.0, 1.0, (n, 6))
    action[:, :, A_KP] = 1.0
    action[:, :, A_KD] = 1.0
    action[:, :, A_MAXT] = 10.0
    d = rng.uniform(-0.1, 0.1, (n, 6)).astype(np.float32)
    twin_action = action.copy()
    twin_action[:, :, A_POS] -= d  # NaN stays NaN
    obs = np.zeros((n, 6, 5), dtype=np.float32)
    twin_obs = np.zeros((n, 6, 5), dtype=np.float32)
    for _ in range(3):
        _lib().hostsim_encoder_offset_servo_tick(sim.h, n, _p(state), _p(action), _p(d), _p(obs))
        _lib().hostsim_encoder_offset_servo_tick(sim.h, n, _p(twin_state), _p(twin_action), None, _p(twin_obs))
        np.testing.assert_array_equal(state, twin_state)  # get_state: bit for bit
        np.testing.assert_array_equal(obs[:, :, 0], twin_obs[:, :, 0] + d)
        np.testing.assert_array_equal(obs[:, :, 1:], twin_obs[:, :, 1:])


def test_zero_offsets_leave_every_bit():
    rng = np.random.default_rng(12)
    n = 32
    state = rng.normal(0.0, 0.5, (n, _abi.STATE_DIM)).astype(np.float32)
    state[:8, _abi.ST_Q:_abi.ST_Q + 6] = -0.0  # a sum with +0 would turn -0 into +0
    view = state.copy()
    changed = np.zeros(n, dtype=np.int32)
    _lib().hostsim_encoder_offset_view(n, _p(view), _p(np.zeros((n, 6), np.float32)), _p(changed, ip))
    assert view.tobytes() == state.tobytes() and not changed.any()
    d = np.zeros((n, 6), dtype=np.float32)
    d[:, 0] = 0.01  # a leg: the gyropod odometry is unchanged
    _lib().hostsim_encoder_offset_view(n, _p(view), _p(d), _p(changed, ip))
    assert not changed.any()
    np.testing.assert_array_equal(view[:, _abi.ST_Q], state[:, _abi.ST_Q] + np.float32(0.01))
    d[:, 5] = -0.02
    _lib().hostsim_encoder_offset_view(n, _p(view), _p(d), _p(changed, ip))
    assert changed.all()


def test_gyropod_leg_targets_start_at_the_reported_positions_and_decay_to_the_servo_zero():
    rng = np.random.default_rng(13)
    n = 16
    sim = _Sim()
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, _abi.INIT_POS + 2] = 0.6
    init[:, _abi.INIT_QUAT] = 1.0
    init[:, _abi.INIT_Q:_abi.INIT_Q + 6] = rng.uniform(-0.2, 0.2, (n, 6))
    d = rng.uniform(-0.1, 0.1, (n, 6)).astype(np.float32)
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    _lib().hostsim_encoder_offset_reset_robot(sim.h, n, _p(state), _p(init), _p(d))
    plain = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    _lib().hostsim_encoder_offset_reset_robot(sim.h, n, _p(plain), _p(init), None)
    # the reset itself is the same physics; the leg targets are the reported (servo-frame) positions
    lt = slice(_abi.ST_LEG_TARGET, _abi.ST_LEG_TARGET + 4)
    other = np.ones(_abi.STATE_DIM, bool)
    other[lt] = False
    np.testing.assert_array_equal(state[:, other], plain[:, other])
    np.testing.assert_array_equal(state[:, lt], state[:, _abi.ST_Q + np.array(LEGS)] + d[:, LEGS])
    # each tick: target <- target + dt * (0 - target), the servo action carries it, and the joints execute target - d
    alpha = np.float32(sim.P.dt)  # low_pass_filter(cutoff_period=1.0)
    obs6 = np.zeros((n, 6), dtype=np.float32)
    servo = np.zeros((n, 6, 6), dtype=np.float32)
    action = np.zeros((n, 2), dtype=np.float32)
    target = state[:, lt].copy()
    for _ in range(5):
        _lib().hostsim_encoder_offset_gyropod_tick(sim.h, n, _p(state), _p(action), _p(d), _p(obs6), _p(servo))
        target = target + alpha * (np.float32(0.0) - target)
        np.testing.assert_array_equal(state[:, lt], target)
        np.testing.assert_array_equal(servo[:, LEGS, A_POS], target)


def test_gyropod_odometry_reports_the_wheel_offsets():
    rng = np.random.default_rng(14)
    n = 16
    sim, state, _ = _standing(n, rng)
    d = np.zeros((n, 6), dtype=np.float32)
    d[:, [2, 5]] = rng.uniform(-0.1, 0.1, (n, 2))
    twin = state.copy()
    obs, twin_obs = np.zeros((n, 6), np.float32), np.zeros((n, 6), np.float32)
    servo = np.zeros((n, 6, 6), dtype=np.float32)
    action = np.zeros((n, 2), dtype=np.float32)
    _lib().hostsim_encoder_offset_gyropod_tick(sim.h, n, _p(state), _p(action), _p(d), _p(obs), _p(servo))
    _lib().hostsim_encoder_offset_gyropod_tick(sim.h, n, _p(twin), _p(action), None, _p(twin_obs), _p(servo))
    np.testing.assert_array_equal(state, twin)  # the wheels run under velocity control: NaN targets
    model = default_model()
    sr = np.float32((1.0 if model.left_wheeled else -1.0) * model.wheel_radius)
    q2, q5 = state[:, _abi.ST_Q + 2], state[:, _abi.ST_Q + 5]
    np.testing.assert_array_equal(obs[:, 0], np.float32(0.5) * ((q2 + d[:, 2]) - (q5 + d[:, 5])) * sr)
    np.testing.assert_array_equal(twin_obs[:, 0], np.float32(0.5) * (q2 - q5) * sr)
    np.testing.assert_array_equal(obs[:, 1:], twin_obs[:, 1:])
    assert (obs[:, 0] != twin_obs[:, 0]).all()


def _why(spec, limits=1, spine=0, body=0):
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_encoder_offset_spec_error(C.byref(spec), limits, spine, body, buf, 256)
    return buf.value.decode() if r else None


def test_spec_rejections():
    ok = _abi.UpkieEncoderOffset(-0.1, 0.1, 0b011011, 0)
    assert _why(ok) is None
    assert _why(_abi.UpkieEncoderOffset(-0.5, 0.5, ALL, 0)) is None
    assert _why(_abi.UpkieEncoderOffset(0.0, 0.0, 1, 0)) is None
    bad_bound = "set_encoder_offset: both bounds must be finite and within [-0.5, 0.5] radians"
    for lo, hi in ((float("nan"), 0.0), (0.0, float("inf")), (-float("inf"), 0.0), (-0.6, 0.0), (0.0, 0.51)):
        assert _why(_abi.UpkieEncoderOffset(lo, hi, ALL, 0)) == bad_bound, (lo, hi)
    assert _why(_abi.UpkieEncoderOffset(0.1, 0.05, ALL, 0)) == "set_encoder_offset: low <= high required"
    bad_mask = "set_encoder_offset: joint_mask must select joints of bits 0 .. 5, at least one"
    for m in (0, 1 << 6, 0xFFFFFFFF):
        assert _why(_abi.UpkieEncoderOffset(-0.1, 0.1, m, 0)) == bad_mask
    assert _why(ok, limits=0) == ("set_encoder_offset: needs joint_limits != 0 (the offsets run in the "
                                  "observation-delay kernels)")
    assert _why(ok, spine=1) == "set_encoder_offset: spine_mode reports the spine's own servos"
    assert _why(ok, body=1) == "set_encoder_offset: body_contacts has no encoder-offset kernels"


def _family(limits=1, spine=0, body=0, obs_delay=0, mode=0, transport=0):
    buf = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_encoder_offset(limits, spine, body, obs_delay, mode, transport, buf, 256)
    return f, buf.value.decode()


def test_family_choice():
    for mode in range(3):
        for transport in (0, 1):
            assert _family(mode=mode, transport=transport)[0] == FAM_SENSE
            assert _family(mode=mode, transport=transport, obs_delay=1)[0] == FAM_SENSE
    assert _family(transport=2) == (
        -1, "encoder offsets have no in-kernel rollout transport (use upkie_b200_step with compact rows)")
    assert _family(spine=1) == (-1, "encoder offsets: spine_mode reports the spine's own servos")
    assert _family(limits=0) == (-1, "encoder offsets need joint_limits != 0")
    assert _family(body=1) == (-1, "encoder offsets have no body-contact kernels")


def test_python_spec_validation():
    s = encoder_offset_spec(0.05)
    assert (s.low, s.high, s.joint_mask) == (np.float32(-0.05), np.float32(0.05), 0b011011)
    s = encoder_offset_spec((-0.01, 0.02), ["left_wheel", "right_knee"])
    assert (s.low, s.high, s.joint_mask) == (np.float32(-0.01), np.float32(0.02), 0b010100)
    assert encoder_offset_spec(None) is None
    assert encoder_offset_spec((-0.5, 0.5)) is not None
    for bad in ((0.2, 0.1), 0.6, (-1.0, 0.0), float("nan"), (0.0, float("inf")), "x", (0.1, 0.2, 0.3), ("a", 0.1)):
        with pytest.raises(UpkieException, match="encoder_offset"):
            encoder_offset_spec(bad)
    with pytest.raises(UpkieException, match="encoder_offset_joints: unknown joint"):
        encoder_offset_spec(0.01, ["left_elbow"])
    with pytest.raises(UpkieException, match="encoder_offset_joints: at least one joint"):
        encoder_offset_spec(0.01, [])
    for kw, what in (({"spine_mode": True}, "spine_mode"), ({"joint_limits": 0}, "joint_limits"),
                     ({"body_contacts": True}, "body_contacts")):
        with pytest.raises(UpkieException, match=f"encoder_offset: .*{what}"):
            encoder_offset_spec(0.01, **kw)
