# SPDX-License-Identifier: Apache-2.0
"""Servo torque scales (upkie_b200_set_torque_scale): the C struct against its mirror; the draw law and the reset
compiled for the CPU (tests/hostsim/torque_scale.cpp) against a NumPy statement of include/upkie_b200.h; servo ticks
against a twin without the spec that is fed the scaled torque (the physics integrates fl(s t), the replies keep t,
external forces come after the scale, a reset's zero-torque substeps stay zero); a unit scale against the twin; the
family the host picks with scales set; the spec's and the state's validation on both sides. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import torque_scale_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
SEED = 0x75CA1E
ALL = 0x3F
WHEELS = 0b100100
A_POS, A_VEL, A_FF, A_KP, A_KD, A_MAXT = (_abi.ACT_KEYS.index(k) for k in (
    "position", "velocity", "feedforward_torque", "kp_scale", "kd_scale", "maximum_torque"))
TAU_MAX = np.asarray(default_model().tau_max, dtype=np.float32)
TORQUE_COLS = list(range(_abi.ST_TORQUE, _abi.ST_TORQUE + 6))

_LIB = None
fp, u32p = C.POINTER(C.c_float), C.POINTER(C.c_uint32)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "torque_scale.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_tscale_"), "libhostsim_torque_scale.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        spec_p = C.POINTER(_abi.UpkieTorqueScale)
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_reset.argtypes = [vp, C.c_int, fp, fp, fp, fp]
        L.hostsim_torque_scale_draw.argtypes = [spec_p, C.c_uint64, C.c_uint64, C.c_uint32, fp]
        L.hostsim_torque_scale_reset.argtypes = [C.c_int, spec_p, C.c_uint64, C.c_uint64, u32p, fp]
        L.hostsim_torque_scale_servo_tick.argtypes = [vp, C.c_int, fp, fp, spec_p, fp, fp, C.c_int, fp]
        L.hostsim_torque_scale_apply.argtypes = [C.c_int, fp, fp, fp]
        L.hostsim_torque_scale_spec_error.argtypes = [spec_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_torque_scale_state_error.argtypes = [C.c_uint32, fp, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_step_family_torque_scale.argtypes = [C.c_int] * 5 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return None if a is None else a.ctypes.data_as(t)


def make_spec(low, high, mask):
    s = _abi.UpkieTorqueScale()
    s.scale_low[:] = list(np.broadcast_to(np.float32(low), 6))
    s.scale_high[:] = list(np.broadcast_to(np.float32(high), 6))
    s.joint_mask = mask
    return s


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def scales_np(spec, seed, g, k):
    """[len(g), 6] the scales of draw k of the envs of global index g (include/upkie_b200.h): fp32, the product
    rounded on its own, clamped to high; exactly 1 outside the mask"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    kk = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4)
    lo = np.asarray(spec.scale_low, dtype=np.float32)
    hi = np.asarray(spec.scale_high, dtype=np.float32)
    out = np.ones(g.shape + (6,), dtype=np.float32)
    for b in range(2):
        w = philox_np(g, np.uint64(1 << 50) | kk | np.uint64(b), np.full(g.shape, seed, dtype=np.uint64))
        for r in range(4):
            j = 4 * b + r
            if j < 6 and (spec.joint_mask >> j) & 1:
                out[:, j] = np.minimum(lo[j] + (hi[j] - lo[j]) * u01(w[r]), hi[j])
    return out


class _Sim:
    def __init__(self, config=None):
        self._m = default_model().to_struct()
        self._c = config if config is not None else _abi.default_sim_config()
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h

    def __del__(self):
        try:
            _lib().hostsim_destroy(self.h)
        except Exception:
            pass

    def tick(self, state, action, spec=None, scale=None, ext=None, zero_torque=False):
        """one servo tick in place; returns the [n, 6, 5] rows"""
        n = state.shape[0]
        obs = np.zeros((n, 6, 5), dtype=np.float32)
        sc = None if scale is None else np.ascontiguousarray(scale.T, dtype=np.float32)  # [6][n]
        ex = None if ext is None else np.ascontiguousarray(ext, dtype=np.float32)
        _lib().hostsim_torque_scale_servo_tick(self.h, n, _p(state), _p(np.ascontiguousarray(action)),
                                               None if spec is None else C.byref(spec), _p(sc), _p(ex),
                                               int(zero_torque), _p(obs))
        return obs


def _standing(n, seed=0):
    """robots dropped onto the floor with small random tilts and joint angles"""
    rng = np.random.default_rng(seed)
    sim = _Sim()
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, _abi.INIT_POS + 2] = 0.58
    pitch = rng.uniform(-0.3, 0.3, n)
    init[:, _abi.INIT_QUAT] = np.cos(pitch / 2)
    init[:, _abi.INIT_QUAT + 2] = np.sin(pitch / 2)
    init[:, _abi.INIT_Q:_abi.INIT_Q + 6] = rng.uniform(-0.3, 0.3, (n, 6))
    _lib().hostsim_reset(sim.h, n, _p(state), _p(init), None, None)
    return sim, state


def _ff_action(ff):
    """feedforward-only commands: no position target, zero gains, the model's effort limit"""
    n = ff.shape[0]
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, A_POS] = np.nan
    a[:, :, A_FF] = ff
    a[:, :, A_MAXT] = TAU_MAX
    return a


def _pd_action(rng, n):
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, A_POS] = rng.uniform(-0.5, 0.5, (n, 6))
    a[:, [2, 5], A_POS] = np.nan
    a[:, :, A_VEL] = rng.uniform(-2.0, 2.0, (n, 6))
    a[:, :, A_FF] = rng.uniform(-1.0, 1.0, (n, 6))
    a[:, :, A_KP] = rng.uniform(0.5, 2.0, (n, 6))
    a[:, :, A_KD] = rng.uniform(0.5, 2.0, (n, 6))
    a[:, :, A_MAXT] = TAU_MAX
    return a


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieTorqueScale \{(.*?)\} UpkieTorqueScale;", header, re.S).group(1)
    names = re.findall(r"\b(\w+)(?:\[\d+\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _abi.UpkieTorqueScale._fields_]
    assert C.sizeof(_abi.UpkieTorqueScale) == 56


@pytest.mark.parametrize("mask", [ALL, WHEELS, 0b011011, 0b010000])
def test_draws_match_the_numpy_law(mask):
    spec = make_spec([0.8, 0.9, 0.7, 0.85, 0.95, 0.75], [1.2, 1.1, 1.3, 1.15, 1.05, 1.25], mask)
    g = np.arange(3, 67, dtype=np.uint64)
    s = np.zeros(6, dtype=np.float32)
    inside = [(mask >> j) & 1 == 1 for j in range(6)]
    for k in (1, 2, 999, 2 ** 31 + 5):
        ref = scales_np(spec, SEED, g, k)
        got = np.zeros((len(g), 6), dtype=np.float32)
        for i, x in enumerate(g):
            _lib().hostsim_torque_scale_draw(C.byref(spec), SEED, int(x), k, _p(s))
            got[i] = s
        np.testing.assert_array_equal(got, ref)
        lo = np.asarray(spec.scale_low, np.float32)
        hi = np.asarray(spec.scale_high, np.float32)
        assert (got[:, inside] >= lo[inside]).all() and (got[:, inside] <= hi[inside]).all()
        assert (got[:, [not x for x in inside]] == np.float32(1.0)).all()  # exactly 1 outside the mask
        for j in range(6):  # both counters of a draw vary across envs
            if inside[j]:
                assert len(np.unique(got[:, j])) == len(g)
    # a mask changes no other joint's draw
    full = scales_np(make_spec(spec.scale_low, spec.scale_high, ALL), SEED, g, 7)
    keep = [j for j in range(6) if inside[j]]
    np.testing.assert_array_equal(scales_np(spec, SEED, g, 7)[:, keep], full[:, keep])


def test_degenerate_range_is_that_scale_and_the_rest_is_one():
    spec = make_spec([0.9, 1.0, 1.25, 0.5, 2.0, 0.75], [0.9, 1.0, 1.25, 0.5, 2.0, 0.75], 0b110111)
    s = np.zeros(6, dtype=np.float32)
    _lib().hostsim_torque_scale_draw(C.byref(spec), SEED, 5, 11, _p(s))
    np.testing.assert_array_equal(s, np.float32([0.9, 1.0, 1.25, 1.0, 2.0, 0.75]))
    assert s.view(np.uint32)[3] == np.float32(1.0).view(np.uint32)


def test_reset_counts_and_stores_the_draw():
    n = 48
    spec = make_spec(0.8, 1.2, 0b101101)
    count = np.full(n, 2, dtype=np.uint32)
    scale = np.zeros((6, n), dtype=np.float32)
    _lib().hostsim_torque_scale_reset(n, C.byref(spec), SEED, 200, _p(count, u32p), _p(scale))
    assert (count == 3).all()
    np.testing.assert_array_equal(scale.T, scales_np(spec, SEED, 200 + np.arange(n), 3))
    # sharding: the draw is keyed on the global env index
    np.testing.assert_array_equal(scale.T[16:], scales_np(spec, SEED, 216 + np.arange(n - 16), 3))


def test_apply_is_one_rounded_product():
    rng = np.random.default_rng(4)
    s = rng.uniform(0.5, 2.0, 4096).astype(np.float32)
    t = rng.uniform(-16.0, 16.0, 4096).astype(np.float32)
    t[:4] = [0.0, -0.0, 16.0, -16.0]
    out = np.empty_like(t)
    _lib().hostsim_torque_scale_apply(t.size, _p(s), _p(t), _p(out))
    assert out.tobytes() == (s * t).tobytes()


@pytest.mark.parametrize("mask", [ALL, WHEELS, 0b011011])
def test_physics_integrates_the_scaled_torque_and_replies_report_the_servos(mask):
    n = 24
    rng = np.random.default_rng(7)
    sim, state = _standing(n, seed=1)
    twin = state.copy()
    spec = make_spec(0.8, 1.2, mask)
    scale = scales_np(spec, SEED, np.arange(n), 1)
    assert (scale[:, [j for j in range(6) if (mask >> j) & 1]] != 1).all()
    start = state.copy()
    for _ in range(30):
        ff = (rng.uniform(-0.5, 0.5, (n, 6)) * TAU_MAX).astype(np.float32)
        obs = sim.tick(state, _ff_action(ff), spec, scale)
        tobs = sim.tick(twin, _ff_action(scale * ff))  # fl(s * tau) in float32
        keep = [c for c in range(_abi.STATE_DIM) if c not in TORQUE_COLS]
        assert state[:, keep].tobytes() == twin[:, keep].tobytes()
        np.testing.assert_array_equal(state[:, TORQUE_COLS], ff)  # the servo's t
        np.testing.assert_array_equal(twin[:, TORQUE_COLS], scale * ff)
        np.testing.assert_array_equal(obs[:, :, 2], ff)
        assert obs[:, :, :2].tobytes() == tobs[:, :, :2].tobytes()
    assert not np.array_equal(state[:, _abi.ST_QD:_abi.ST_QD + 6], start[:, _abi.ST_QD:_abi.ST_QD + 6])  # it moved


def test_external_forces_are_added_after_the_scale():
    n = 16
    rng = np.random.default_rng(8)
    sim, state = _standing(n, seed=2)
    twin = state.copy()
    spec = make_spec(0.8, 1.2, ALL)
    scale = scales_np(spec, SEED, np.arange(n), 4)
    ext = rng.uniform(-30.0, 30.0, (n, 7, 3)).astype(np.float32)
    for _ in range(10):
        ff = (rng.uniform(-0.5, 0.5, (n, 6)) * TAU_MAX).astype(np.float32)
        sim.tick(state, _ff_action(ff), spec, scale, ext=ext)
        sim.tick(twin, _ff_action(scale * ff), ext=ext)
        keep = [c for c in range(_abi.STATE_DIM) if c not in TORQUE_COLS]
        assert state[:, keep].tobytes() == twin[:, keep].tobytes()


def test_zero_torque_substeps_stay_zero():
    n = 16
    rng = np.random.default_rng(9)
    sim, state = _standing(n, seed=3)
    twin = state.copy()
    spec = make_spec(0.5, 2.0, ALL)
    scale = scales_np(spec, SEED, np.arange(n), 2)
    action = _pd_action(rng, n)
    obs = sim.tick(state, action, spec, scale, zero_torque=True)
    tobs = sim.tick(twin, action, zero_torque=True)
    assert state.tobytes() == twin.tobytes() and obs.tobytes() == tobs.tobytes()


def test_unit_scale_leaves_every_bit():
    n = 32
    rng = np.random.default_rng(10)
    cfg = _abi.default_sim_config()
    for j in range(6):
        cfg.joint_friction[j] = 0.3  # friction folded into the command, scaled with it
    sim = _Sim(cfg)
    _, state = _standing(n, seed=4)
    twin = state.copy()
    spec = make_spec(1.0, 1.0, ALL)
    scale = np.ones((n, 6), dtype=np.float32)
    for _ in range(8):
        action = _pd_action(rng, n)
        obs = sim.tick(state, action, spec, scale)
        tobs = sim.tick(twin, action)
        assert state.tobytes() == twin.tobytes() and obs.tobytes() == tobs.tobytes()


def _why(spec, limits=1, spine=0, body=0):
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_torque_scale_spec_error(C.byref(spec), limits, spine, body, buf, 256)
    return buf.value.decode() if r else None


def test_spec_rejections():
    ok = make_spec(0.8, 1.2, 0b011011)
    assert _why(ok) is None
    assert _why(make_spec(2.0, 2.0, ALL)) is None
    assert _why(make_spec(1e-6, 1e-6, ALL)) is None
    # joints outside the mask may hold any finite values
    assert _why(make_spec([0.0, 0.9, -1.0, 0.9, 0.9, 0.9], [0.0, 1.1, 5.0, 1.1, 1.1, 1.1], 0b111010)) is None
    finite = "set_torque_scale: every bound must be finite"
    for field in ("scale_low", "scale_high"):
        for x in (float("nan"), float("inf"), -float("inf")):
            s = make_spec(0.8, 1.2, WHEELS)
            getattr(s, field)[0] = x  # a joint outside the mask too
            assert _why(s) == finite, (field, x)
    rng = "set_torque_scale: 0 < scale_low <= scale_high <= 2 required on every joint of the mask"
    for lo, hi in ((0.0, 1.0), (-0.5, 1.0), (1.2, 0.8), (0.9, 2.0001), (2.5, 3.0)):
        assert _why(make_spec(lo, hi, ALL)) == rng, (lo, hi)
    bad_mask = "set_torque_scale: joint_mask must select joints of bits 0 .. 5, at least one"
    for m in (0, 1 << 6, 0xFFFFFFFF):
        assert _why(make_spec(0.8, 1.2, m)) == bad_mask
    s = make_spec(0.8, 1.2, ALL)
    s.reserved = 1
    assert _why(s) == "set_torque_scale: reserved must be 0"
    assert _why(ok, limits=0) == ("set_torque_scale: needs joint_limits != 0 (the scale runs in the "
                                  "observation-delay kernels)")
    assert _why(ok, spine=1) == "set_torque_scale: spine_mode applies the spine's own torque law"
    assert _why(ok, body=1) == "set_torque_scale: body_contacts has no torque-scale kernels"


def _state_why(mask, v):
    v = np.ascontiguousarray(v, dtype=np.float32)
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_torque_scale_state_error(mask, _p(v), v.shape[0], buf, 256)
    return buf.value.decode() if r else None


def test_state_rejections():
    n = 5
    good = np.ones((n, 6), dtype=np.float32)
    good[:, [2, 5]] = [[0.5, 2.0]] * n
    assert _state_why(WHEELS, good) is None
    inside = "set_torque_scale_state: every scale of a joint of joint_mask must be in (0, 2]"
    for x in (0.0, -0.0, -1.0, 2.0001, float("nan"), float("inf")):
        v = good.copy()
        v[3, 5] = x
        assert _state_why(WHEELS, v) == inside, x
    outside = "set_torque_scale_state: a joint outside joint_mask must have a scale of exactly 1"
    for x in (0.9, np.nextafter(np.float32(1), np.float32(2)), 0.0, float("nan")):
        v = good.copy()
        v[1, 0] = x
        assert _state_why(WHEELS, v) == outside, x


def _family(limits=1, spine=0, body=0, mode=0, transport=0):
    buf = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_torque_scale(limits, spine, body, mode, transport, buf, 256)
    return f, buf.value.decode()


def test_family_choice():
    for mode in range(3):
        for transport in (0, 1):
            assert _family(mode=mode, transport=transport)[0] == FAM_SENSE
    assert _family(transport=2) == (
        -1, "torque scales have no in-kernel rollout transport (use upkie_b200_step with compact rows)")
    assert _family(spine=1) == (-1, "torque scales: spine_mode applies the spine's own torque law")
    assert _family(limits=0) == (-1, "torque scales need joint_limits != 0")
    assert _family(body=1) == (-1, "torque scales have no body-contact kernels")


def test_python_spec_validation():
    s = torque_scale_spec((0.9, 1.1))
    assert s.joint_mask == ALL
    np.testing.assert_array_equal(s.scale_low, np.float32(0.9))
    np.testing.assert_array_equal(s.scale_high, np.float32(1.1))
    s = torque_scale_spec(0.95, ["left_wheel", "right_wheel"])
    assert s.joint_mask == WHEELS and s.scale_low[2] == np.float32(0.95) and s.scale_high[5] == np.float32(0.95)
    s = torque_scale_spec({"left_knee": (0.8, 1.2), "right_wheel": 1.5})
    assert s.joint_mask == 0b100010
    assert (s.scale_low[1], s.scale_high[1], s.scale_low[5]) == (np.float32(0.8), np.float32(1.2), 1.5)
    assert s.scale_low[0] == 1.0 and s.scale_high[0] == 1.0
    assert _why(s) is None
    assert torque_scale_spec(None) is None
    for bad in ((1.2, 0.8), 0.0, (-1.0, 1.0), (0.5, 2.5), float("nan"), (0.9, float("inf")), "x", (0.9, 1.0, 1.1),
                {"left_knee": (1.1, 0.9)}, {"left_knee": "x"}):
        with pytest.raises(UpkieException, match="torque_scale"):
            torque_scale_spec(bad)
    with pytest.raises(UpkieException, match="unknown joint"):
        torque_scale_spec(1.0, ["left_elbow"])
    with pytest.raises(UpkieException, match="unknown joint"):
        torque_scale_spec({"left_elbow": 1.0})
    with pytest.raises(UpkieException, match="has no scale"):
        torque_scale_spec({"left_knee": 1.0}, ["left_hip"])
    with pytest.raises(UpkieException, match="at least one joint"):
        torque_scale_spec(1.0, [])
    for kw, what in (({"spine_mode": True}, "spine_mode"), ({"joint_limits": 0}, "joint_limits"),
                     ({"body_contacts": True}, "body_contacts")):
        with pytest.raises(UpkieException, match=f"torque_scale: .*{what}"):
            torque_scale_spec((0.9, 1.1), **kw)
