# SPDX-License-Identifier: Apache-2.0
"""Servo velocity limits (upkie_b200_set_velocity_derate): the C struct against its mirror; the draw law and the reset
compiled for the CPU (tests/hostsim/velocity_derate.cpp) against a NumPy statement of include/upkie_b200.h; the torque
law against a float32 NumPy restatement; a servo tick whose limits no joint reaches against its twin without them; a
free-spinning wheel under full torque; the family the host picks with limits set; the spec's validation on both sides.
No GPU needed."""
import ctypes as C
import math
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import UPKIE_VELOCITY_DERATE, velocity_derate_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
SEED = 0x7E10C
ALL = 0x3F
WHEELS = 0b100100
A_POS, A_VEL, A_FF, A_KP, A_KD, A_MAXT = (_abi.ACT_KEYS.index(k) for k in (
    "position", "velocity", "feedforward_torque", "kp_scale", "kd_scale", "maximum_torque"))
TAU_MAX = np.asarray(default_model().tau_max, dtype=np.float32)

_LIB = None
fp, u32p = C.POINTER(C.c_float), C.POINTER(C.c_uint32)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "velocity_derate.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_vlim_"), "libhostsim_velocity_derate.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        spec_p = C.POINTER(_abi.UpkieVelocityDerate)
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_reset.argtypes = [vp, C.c_int, fp, fp, fp, fp]
        L.hostsim_velocity_derate_draw.argtypes = [spec_p, C.c_uint64, C.c_uint64, C.c_uint32, fp]
        L.hostsim_velocity_derate_reset.argtypes = [C.c_int, spec_p, C.c_uint64, C.c_uint64, u32p, fp]
        L.hostsim_velocity_derate_torque.argtypes = [C.c_int, fp, fp, fp, fp, fp, fp]
        L.hostsim_velocity_derate_servo_tick.argtypes = [vp, C.c_int, fp, fp, spec_p, fp, fp, fp]
        L.hostsim_velocity_derate_spec_error.argtypes = [spec_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_step_family_velocity_derate.argtypes = [C.c_int] * 5 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return None if a is None else a.ctypes.data_as(t)


def make_spec(low, high, derate, mask):
    s = _abi.UpkieVelocityDerate()
    s.max_velocity_low[:] = list(np.broadcast_to(np.float32(low), 6))
    s.max_velocity_high[:] = list(np.broadcast_to(np.float32(high), 6))
    s.derate[:] = list(np.broadcast_to(np.float32(derate), 6))
    s.joint_mask = mask
    return s


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def limits_np(spec, seed, g, k):
    """[len(g), 6] the limits of draw k of the envs of global index g (include/upkie_b200.h): fp32, the product
    rounded on its own, clamped to high; exactly 0 outside the mask"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    kk = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4)
    lo = np.asarray(spec.max_velocity_low, dtype=np.float32)
    hi = np.asarray(spec.max_velocity_high, dtype=np.float32)
    out = np.zeros(g.shape + (6,), dtype=np.float32)
    for b in range(2):
        w = philox_np(g, np.uint64(1 << 52) | kk | np.uint64(b), np.full(g.shape, seed, dtype=np.uint64))
        for r in range(4):
            j = 4 * b + r
            if j < 6 and (spec.joint_mask >> j) & 1:
                out[:, j] = np.minimum(lo[j] + (hi[j] - lo[j]) * u01(w[r]), hi[j])
    return out


def law_np(t, qd, v, derate, tau_max):
    """The derate law of include/upkie_b200.h in float32: past |qd| > v, the torque driving the joint faster is capped
    by clip((v + derate - |qd|) / derate, 0, 1) * tau_max; anything else is t"""
    t, qd, v, derate, tau_max = (np.asarray(x, dtype=np.float32) for x in (t, qd, v, derate, tau_max))
    s = np.abs(qd)
    cap = np.clip(((v + derate) - s) / derate, np.float32(0), np.float32(1)) * tau_max
    return np.where(s > v, np.where(qd > 0, np.fmin(t, cap), np.fmax(t, -cap)), t).astype(np.float32)


class _Sim:
    def __init__(self, config=None):
        self._m = default_model().to_struct()
        self._c = config if config is not None else _abi.default_sim_config()
        self.P = self._c
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h

    def __del__(self):
        try:
            _lib().hostsim_destroy(self.h)
        except Exception:
            pass

    def tick(self, state, action, spec=None, vmax=None):
        """one servo tick in place; returns the [n, 6, 5] rows and the largest |qd| of each joint over the substeps"""
        n = state.shape[0]
        obs = np.zeros((n, 6, 5), dtype=np.float32)
        peak = np.zeros((n, 6), dtype=np.float32)
        vm = None if vmax is None else np.ascontiguousarray(vmax.T, dtype=np.float32)  # [6][n]
        _lib().hostsim_velocity_derate_servo_tick(self.h, n, _p(state), _p(np.ascontiguousarray(action)),
                                                  None if spec is None else C.byref(spec), _p(vm), _p(obs), _p(peak))
        return obs, peak


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieVelocityDerate \{(.*?)\} UpkieVelocityDerate;", header, re.S).group(1)
    names = re.findall(r"\b(\w+)(?:\[\d+\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _abi.UpkieVelocityDerate._fields_]
    assert C.sizeof(_abi.UpkieVelocityDerate) == 80


@pytest.mark.parametrize("mask", [ALL, WHEELS, 0b011011, 0b010000])
def test_draws_match_the_numpy_law(mask):
    spec = make_spec([10.0, 11.0, 40.0, 12.0, 13.0, 45.0], [14.0, 15.0, 55.0, 16.0, 17.0, 60.0], 12.0, mask)
    g = np.arange(3, 67, dtype=np.uint64)
    v = np.zeros(6, dtype=np.float32)
    inside = [(mask >> j) & 1 == 1 for j in range(6)]
    for k in (1, 2, 999, 2 ** 31 + 5):
        ref = limits_np(spec, SEED, g, k)
        got = np.zeros((len(g), 6), dtype=np.float32)
        for i, x in enumerate(g):
            _lib().hostsim_velocity_derate_draw(C.byref(spec), SEED, int(x), k, _p(v))
            got[i] = v
        np.testing.assert_array_equal(got, ref)
        lo = np.asarray(spec.max_velocity_low, np.float32)
        hi = np.asarray(spec.max_velocity_high, np.float32)
        assert (got[:, inside] >= lo[inside]).all() and (got[:, inside] <= hi[inside]).all()
        out = got[:, [not x for x in inside]]
        assert (out == 0).all() and not np.signbit(out).any()  # exactly +0 outside the mask
        for j in range(6):  # both counters of a draw vary across envs
            if inside[j]:
                assert len(np.unique(got[:, j])) == len(g)
    # a mask changes no other joint's draw
    full = limits_np(make_spec(spec.max_velocity_low, spec.max_velocity_high, 12.0, ALL), SEED, g, 7)
    keep = [j for j in range(6) if inside[j]]
    np.testing.assert_array_equal(limits_np(spec, SEED, g, 7)[:, keep], full[:, keep])


def test_degenerate_range_is_that_limit():
    spec = make_spec(12.5, 12.5, 4.0, ALL)
    v = np.zeros(6, dtype=np.float32)
    _lib().hostsim_velocity_derate_draw(C.byref(spec), SEED, 5, 11, _p(v))
    np.testing.assert_array_equal(v, np.float32(12.5))


def test_reset_counts_and_stores_the_draw():
    n = 48
    spec = make_spec(8.0, 20.0, 5.0, 0b101101)
    count = np.full(n, 2, dtype=np.uint32)
    vmax = np.zeros((6, n), dtype=np.float32)
    _lib().hostsim_velocity_derate_reset(n, C.byref(spec), SEED, 200, _p(count, u32p), _p(vmax))
    assert (count == 3).all()
    np.testing.assert_array_equal(vmax.T, limits_np(spec, SEED, 200 + np.arange(n), 3))
    # sharding: the draw is keyed on the global env index
    np.testing.assert_array_equal(vmax.T[16:], limits_np(spec, SEED, 216 + np.arange(n - 16), 3))


def _law_c(t, qd, v, derate, tau_max):
    arrs = [np.ascontiguousarray(np.broadcast_to(np.asarray(x, np.float32), np.shape(t))) for x in
            (t, qd, v, derate, tau_max)]
    out = np.empty(np.shape(t), dtype=np.float32)
    _lib().hostsim_velocity_derate_torque(out.size, *(_p(a) for a in arrs), _p(out))
    return out


def test_law_matches_the_numpy_restatement_on_a_grid():
    v, d = np.float32(12.566371), np.float32(12.566371)
    speeds = np.array([0.0, 1.0, 12.0, 12.566371, 12.566372, 13.0, 18.0, 25.0, 25.132742, 26.0, 60.0, 100.0],
                      dtype=np.float32)
    qd = np.concatenate([speeds, -speeds, [np.float32(-0.0)]]).astype(np.float32)
    # torques of the servo law: full motoring and braking, partial, and commands with a reduced maximum_torque (the
    # law clips first, the derate caps with the model's effort limit)
    t = np.array([16.0, -16.0, 3.0, -3.0, 0.0, -0.0, 0.5, -0.5, 15.999, -7.25], dtype=np.float32)
    T, Q = np.meshgrid(t, qd, indexing="ij")
    got = _law_c(T, Q, v, d, np.float32(16.0))
    ref = law_np(T, Q, v, d, np.float32(16.0))
    assert got.tobytes() == ref.tobytes()
    below = np.abs(Q) <= v
    braking = T * Q < 0
    unchanged = below | braking
    assert got[unchanged].tobytes() == T[unchanged].tobytes()  # bit for bit, -0 included
    assert (got[T == 0] == 0).all()  # a zero torque stays zero (of either sign)
    # past the band, no torque drives the joint faster
    past = np.abs(Q) >= v + d
    assert (got[past & (Q > 0)] <= 0).all() and (got[past & (Q < 0)] >= 0).all()
    # inside the band the cap falls linearly
    q = np.float32(18.0)
    assert got[0, list(qd).index(q)] == np.float32((v + d - q) / d) * np.float32(16.0)
    assert got[1, list(qd).index(q)] == np.float32(-16.0)  # braking


def _free_wheel_state(n, gravity=0.0):
    """robots floating clear of the floor (gravity 0): the wheels spin freely"""
    cfg = _abi.default_sim_config()
    cfg.gravity = gravity
    sim = _Sim(cfg)
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, _abi.INIT_POS + 2] = 1.2
    init[:, _abi.INIT_QUAT] = 1.0
    _lib().hostsim_reset(sim.h, n, _p(state), _p(init), None, None)
    return sim, state


def _wheel_action(n, sign):
    """legs held at zero, wheels under pure feedforward sign * tau_max"""
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, A_KP] = 1.0
    a[:, :, A_KD] = 1.0
    a[:, :, A_MAXT] = TAU_MAX
    for w in (2, 5):
        a[:, w, A_POS] = np.nan
        a[:, w, A_KP] = 0.0
        a[:, w, A_KD] = 0.0
        a[:, w, A_FF] = sign * TAU_MAX[w]
    return a


def test_limits_no_joint_reaches_leave_every_bit():
    # limits above max_coordinate_velocity: no joint ever passes them
    rng = np.random.default_rng(21)
    n = 32
    sim, state = _free_wheel_state(n, gravity=9.81)
    state[:, _abi.ST_POS + 2] = 0.6
    twin = state.copy()
    action = _wheel_action(n, 1.0)
    action[:, :, A_POS] = np.where(np.isnan(action[:, :, A_POS]), np.nan, rng.uniform(-0.3, 0.3, (n, 6)))
    spec = make_spec(150.0, 200.0, 10.0, ALL)
    vmax = np.tile(np.float32(150.0), (n, 6))
    for _ in range(6):
        obs, _ = sim.tick(state, action, spec, vmax)
        tobs, _ = sim.tick(twin, action)
        assert state.tobytes() == twin.tobytes()
        assert obs.tobytes() == tobs.tobytes()


def test_free_wheel_saturates_within_its_band():
    n = 8
    sim, state = _free_wheel_state(n)
    twin = state.copy()
    v = np.linspace(15.0, 40.0, n).astype(np.float32)
    derate = np.float32(10.0)
    spec = make_spec(1.0, 100.0, derate, WHEELS)
    vmax = np.zeros((n, 6), dtype=np.float32)
    vmax[:, 2] = vmax[:, 5] = v
    action = _wheel_action(n, 1.0)
    model = default_model()
    i_wheel = float(np.asarray(model.inertia)[3][1])  # about the wheel axis (y)
    h = np.float32(1.0 / (200.0 * 5))
    bound = v + derate + np.float32(TAU_MAX[2]) * h / np.float32(i_wheel)
    peak = np.zeros((n, 6), dtype=np.float32)
    tpeak = np.zeros((n, 6), dtype=np.float32)
    for _ in range(40):
        _, p = sim.tick(state, action, spec, vmax)
        _, tp = sim.tick(twin, action)
        peak = np.maximum(peak, p)
        tpeak = np.maximum(tpeak, tp)
    for w in (2, 5):
        assert (peak[:, w] <= bound).all(), (peak[:, w], bound)
        assert (peak[:, w] > v).all()  # the wheel does pass its limit
        assert (tpeak[:, w] > bound).all()  # its twin without the spec does not stop there
    # a reversed command from above the band brakes exactly as the twin: a braking torque passes unchanged
    fast = twin.copy()
    assert (np.abs(fast[:, _abi.ST_QD + 2]) > v + derate).all()
    braked, braked_twin = fast.copy(), fast.copy()
    back = _wheel_action(n, -1.0)
    for _ in range(3):
        obs, _ = sim.tick(braked, back, spec, vmax)
        tobs, _ = sim.tick(braked_twin, back)
        assert braked.tobytes() == braked_twin.tobytes()
        assert obs.tobytes() == tobs.tobytes()
    assert (braked[:, _abi.ST_QD + 2] > 0).all()  # still spinning forward: every substep braked


def _why(spec, limits=1, spine=0, body=0):
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_velocity_derate_spec_error(C.byref(spec), limits, spine, body, buf, 256)
    return buf.value.decode() if r else None


def test_spec_rejections():
    ok = make_spec(10.0, 20.0, 5.0, 0b011011)
    assert _why(ok) is None
    assert _why(make_spec(10.0, 10.0, 1e-3, ALL)) is None
    # joints outside the mask may hold any finite values
    assert _why(make_spec([0.0, 5.0, -1.0, 5.0, 5.0, 5.0], [0.0, 6.0, -2.0, 6.0, 6.0, 6.0],
                          [0.0, 1.0, -1.0, 1.0, 1.0, 1.0], 0b111010)) is None
    finite = "set_velocity_derate: every bound must be finite"
    for field in ("max_velocity_low", "max_velocity_high", "derate"):
        for x in (float("nan"), float("inf"), -float("inf")):
            s = make_spec(10.0, 20.0, 5.0, WHEELS)
            getattr(s, field)[0] = x  # a joint outside the mask too
            assert _why(s) == finite, (field, x)
    rng = "set_velocity_derate: 0 < max_velocity_low <= max_velocity_high required on every joint of the mask"
    for lo, hi in ((0.0, 10.0), (-1.0, 10.0), (20.0, 10.0)):
        assert _why(make_spec(lo, hi, 5.0, ALL)) == rng
    for d in (0.0, -1.0):
        assert _why(make_spec(10.0, 20.0, d, ALL)) == "set_velocity_derate: derate > 0 required on every joint of the mask"
    bad_mask = "set_velocity_derate: joint_mask must select joints of bits 0 .. 5, at least one"
    for m in (0, 1 << 6, 0xFFFFFFFF):
        assert _why(make_spec(10.0, 20.0, 5.0, m)) == bad_mask
    s = make_spec(10.0, 20.0, 5.0, ALL)
    s.reserved = 1
    assert _why(s) == "set_velocity_derate: reserved must be 0"
    assert _why(ok, limits=0) == ("set_velocity_derate: needs joint_limits != 0 (the limits run in the "
                                  "observation-delay kernels)")
    assert _why(ok, spine=1) == "set_velocity_derate: spine_mode applies the spine's own torque law"
    assert _why(ok, body=1) == "set_velocity_derate: body_contacts has no velocity-limit kernels"


def _family(limits=1, spine=0, body=0, mode=0, transport=0):
    buf = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_velocity_derate(limits, spine, body, mode, transport, buf, 256)
    return f, buf.value.decode()


def test_family_choice():
    for mode in range(3):
        for transport in (0, 1):
            assert _family(mode=mode, transport=transport)[0] == FAM_SENSE
    assert _family(transport=2) == (
        -1, "velocity limits have no in-kernel rollout transport (use upkie_b200_step with compact rows)")
    assert _family(spine=1) == (-1, "velocity limits: spine_mode applies the spine's own torque law")
    assert _family(limits=0) == (-1, "velocity limits need joint_limits != 0")
    assert _family(body=1) == (-1, "velocity limits have no body-contact kernels")


def test_upkie_preset_is_the_configured_robot():
    rev = 2.0 * math.pi
    s = velocity_derate_spec(UPKIE_VELOCITY_DERATE)
    assert s.joint_mask == ALL
    np.testing.assert_array_equal(s.max_velocity_low, np.float32([2 * rev, 2 * rev, 8 * rev, 2 * rev, 2 * rev, 8 * rev]))
    np.testing.assert_array_equal(s.max_velocity_high, s.max_velocity_low)
    np.testing.assert_array_equal(s.derate, np.float32(2 * rev))
    assert abs(s.max_velocity_low[2] * default_model().wheel_radius - 2.513) < 1e-3  # m/s of ground velocity
    assert _why(s) is None


def test_python_spec_validation():
    s = velocity_derate_spec({"max_velocity": (10.0, 20.0)})
    assert s.joint_mask == ALL and list(s.max_velocity_low) == [10.0] * 6 and list(s.max_velocity_high) == [20.0] * 6
    np.testing.assert_array_equal(s.derate, np.float32(_abi.MOTEUS_MAX_VELOCITY_DERATE))
    s = velocity_derate_spec({"max_velocity": 30.0, "derate": 5.0}, ["left_wheel", "right_wheel"])
    assert s.joint_mask == WHEELS and s.max_velocity_low[2] == 30.0 and s.derate[5] == 5.0
    s = velocity_derate_spec({"max_velocity": {"left_knee": (11.0, 12.0), "right_wheel": 40.0},
                              "derate": {"right_wheel": 3.0}})
    assert s.joint_mask == 0b100010
    assert (s.max_velocity_low[1], s.max_velocity_high[1], s.max_velocity_low[5]) == (11.0, 12.0, 40.0)
    assert s.derate[5] == 3.0 and s.derate[1] == np.float32(_abi.MOTEUS_MAX_VELOCITY_DERATE)
    assert velocity_derate_spec(None) is None
    for bad in ({"max_velocity": (20.0, 10.0)}, {"max_velocity": 0.0}, {"max_velocity": (-1.0, 5.0)},
                {"max_velocity": float("nan")}, {"max_velocity": (1.0, float("inf"))}, {"max_velocity": "x"},
                {"max_velocity": (1.0, 2.0, 3.0)}, {"max_velocity": 10.0, "derate": 0.0},
                {"max_velocity": 10.0, "derate": float("inf")}, {"max_velocity": 10.0, "derate": "x"},
                {"max_velocity": 10.0, "band": 1.0}, {"derate": 1.0}, 10.0, (1.0, 2.0)):
        with pytest.raises(UpkieException, match="velocity_derate"):
            velocity_derate_spec(bad)
    with pytest.raises(UpkieException, match="unknown joint"):
        velocity_derate_spec({"max_velocity": 10.0}, ["left_elbow"])
    with pytest.raises(UpkieException, match="unknown joint"):
        velocity_derate_spec({"max_velocity": {"left_elbow": 10.0}})
    with pytest.raises(UpkieException, match="has no max_velocity"):
        velocity_derate_spec({"max_velocity": {"left_knee": 10.0}}, ["left_hip"])
    with pytest.raises(UpkieException, match="at least one joint"):
        velocity_derate_spec({"max_velocity": 10.0}, [])
    for kw, what in (({"spine_mode": True}, "spine_mode"), ({"joint_limits": 0}, "joint_limits"),
                     ({"body_contacts": True}, "body_contacts")):
        with pytest.raises(UpkieException, match=f"velocity_derate: .*{what}"):
            velocity_derate_spec({"max_velocity": 10.0}, **kw)
