# SPDX-License-Identifier: Apache-2.0
"""Push randomisation (upkie_b200_set_push_randomization): the C struct against its mirror, the draw and the schedule
the kernels run, compiled for the CPU (tests/hostsim/pushes.cpp), against a NumPy statement of the law, the spec's
validation, and the B200VectorEnv dict form. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import push_randomization_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")

# ticks of a schedule (push_schedule_np, hostsim_push_run): a counted step, a next-step reset (the reset substep, not
# counted), a counted step followed by a same-step reset
STEP, NEXT_STEP_RESET, SAME_STEP_RESET = 0, 1, 2


def test_struct_matches_the_header():
    header = open(HEADER).read()
    assert re.search(r"#define UPKIE_PUSH_MAX_STEPS \(1u << (\d+)\)", header).group(1) == "30"
    assert _abi.PUSH_MAX_STEPS == 1 << 30
    body = re.search(r"typedef struct UpkiePushRandomization \{(.*?)\} UpkiePushRandomization;", header, re.S).group(1)
    names = re.findall(r"(\w+)(?:\[\d\])?\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f for f, _ in _abi.UpkiePushRandomization._fields_]
    S = _abi.UpkiePushRandomization
    assert (S.body.offset, S.gap_low.offset, S.duration_high.offset, S.force_low.offset, S.force_high.offset,
            C.sizeof(S)) == (0, 4, 16, 20, 32, 44)


# ---- NumPy statement of the law ----------------------------------------------------------------------------------------


def _tag(k, b):
    return np.uint64(1 << 62) | (np.asarray(k, dtype=np.uint64) << np.uint64(4)) | np.uint64(b)


def push_draw_np(spec, seed, env_index, k):
    """Draw k of the envs of global index env_index (arrays broadcast): (gap, duration) uint32 and force [.., 3] fp32,
    as include/upkie_b200.h states the law"""
    g = np.atleast_1d(np.asarray(env_index, dtype=np.uint64))
    k = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape)
    key = np.full(g.shape, seed, dtype=np.uint64)
    w0 = philox_np(g, _tag(k, 0), key)
    w1 = philox_np(g, _tag(k, 1), key)
    words = [w0[0], w0[1], w0[2], w0[3], w1[0]]

    def steps(w, lo, hi):
        return (np.uint64(lo) + (((w >> np.uint32(8)).astype(np.uint64) * np.uint64(hi - lo + 1)) >> np.uint64(24))
                ).astype(np.uint32)

    gap = steps(words[0], spec.gap_low, spec.gap_high)
    duration = steps(words[1], spec.duration_low, spec.duration_high)
    force = np.empty(g.shape + (3,), dtype=np.float32)
    for a in range(3):
        lo, hi = np.float32(spec.force_low[a]), np.float32(spec.force_high[a])
        u = (words[2 + a] >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)
        force[..., a] = np.minimum(lo + (hi - lo) * u, hi)
    return gap, duration, force


def push_schedule_np(spec, seed, env_index, ticks, count0=0, timer0=0):
    """The schedule of the envs env_index [N] over ticks [T, N] (STEP, NEXT_STEP_RESET or SAME_STEP_RESET):
    applied [T, N, 3] the push each tick's physics took, reported [T, N, 3] what upkie_b200_get_push_forces returns
    after it (zero after a reset), and the state (count, timer) [T, N] after each tick"""
    g = np.atleast_1d(np.asarray(env_index, dtype=np.uint64))
    ticks = np.asarray(ticks).reshape(-1, g.size)
    k = np.broadcast_to(np.asarray(count0, dtype=np.uint64), g.shape).copy()
    t = np.broadcast_to(np.asarray(timer0, dtype=np.uint64), g.shape).copy()
    T = ticks.shape[0]
    applied = np.zeros((T, g.size, 3), dtype=np.float32)
    count, timer = np.zeros((T, g.size), dtype=np.uint32), np.zeros((T, g.size), dtype=np.uint32)
    for s in range(T):
        gap, dur, f = push_draw_np(spec, seed, g, k)
        end = gap.astype(np.uint64) + dur
        reset = ticks[s] == NEXT_STEP_RESET
        # a counted step: a push that ran out at the last one starts the next draw
        roll = ~reset & (t >= end)
        k = np.where(roll, k + 1, k)
        t = np.where(roll, 0, t)
        gap2, dur2, f2 = push_draw_np(spec, seed, g, k)
        gap, f = np.where(roll, gap2, gap), np.where(roll[:, None], f2, f)
        end = np.where(roll, gap2.astype(np.uint64) + dur2, end)
        t = np.where(reset, t, t + 1)
        pushed = ~reset & (t > gap)
        applied[s] = np.where(pushed[:, None], f, np.float32(0))
        # resets: the next draw, after the +1 of a push that ran out
        restart = reset | (ticks[s] == SAME_STEP_RESET)
        k = np.where(restart, k + np.where(t >= end, 2, 1).astype(np.uint64), k)
        t = np.where(restart, 0, t)
        count[s], timer[s] = k, t
    reported = np.where((ticks == STEP)[..., None], applied, np.float32(0))
    return applied, reported, count, timer


# ---- the CPU build of the kernels' code --------------------------------------------------------------------------------

_LIB = None


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "pushes.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_push_"), "libhostsim_push.so")
        # tools/hostsim_sanitizers.sh sets the flags of an AddressSanitizer / UBSan build
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        sp, fp = C.POINTER(_abi.UpkiePushRandomization), C.POINTER(C.c_float)
        u32p, u8p = C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)
        L.hostsim_push_draw.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_uint32, u32p, fp]
        L.hostsim_push_run.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_int, u8p, C.c_uint32, C.c_uint32, fp, u32p,
                                       u32p]
        L.hostsim_push_last_force.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, fp]
        L.hostsim_push_reset.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_int, u8p, u32p, u32p]
        L.hostsim_push_spec_valid.argtypes = [sp]
        _LIB = L
    return _LIB


def _p(a, t):
    return a.ctypes.data_as(C.POINTER(t))


def make_spec(body=0, gap=(3, 9), duration=(1, 4), force=((-40.0, -20.0, 0.0), (40.0, 20.0, 5.0))):
    s = _abi.UpkiePushRandomization()
    s.body = body
    s.gap_low, s.gap_high = gap
    s.duration_low, s.duration_high = duration
    for a in range(3):
        s.force_low[a], s.force_high[a] = force[0][a], force[1][a]
    return s


@pytest.mark.parametrize("seed", [0, 7, 2**40 + 3])
def test_draw_matches_the_numpy_law(seed):
    L = _lib()
    specs = [make_spec(), make_spec(gap=(0, 0), duration=(1, 1)), make_spec(gap=(0, 2**30), duration=(5, 2**30)),
             make_spec(force=((1.5, 1.5, -3.0), (1.5, 2.5, -3.0)))]
    for spec in specs:
        for env in (0, 1, 4095, 65535, 2**33 + 17):
            for k in (0, 1, 2, 3, 1000, 2**32 - 1):
                steps, f = (C.c_uint32 * 2)(), np.empty(3, dtype=np.float32)
                L.hostsim_push_draw(C.byref(spec), seed, env, k, steps, _p(f, C.c_float))
                gap, dur, force = push_draw_np(spec, seed, env, k)
                assert (steps[0], steps[1]) == (gap[0], dur[0])
                np.testing.assert_array_equal(f, force[0])
                assert spec.gap_low <= steps[0] <= spec.gap_high
                assert spec.duration_low <= steps[1] <= spec.duration_high
                assert np.all(f >= np.float32(spec.force_low)) and np.all(f <= np.float32(spec.force_high))


def test_steps_cover_their_range_uniformly():
    spec = make_spec(gap=(2, 5), duration=(1, 3))
    gap, dur, _ = push_draw_np(spec, 3, np.arange(40000), 1)
    for values, lo, hi in ((gap, 2, 5), (dur, 1, 3)):
        counts = np.bincount(values, minlength=hi + 1)[lo:]
        assert counts.size == hi - lo + 1 and np.all(np.abs(counts / values.size - 1 / counts.size) < 0.01)


def _random_ticks(rng, T, n, mode):
    ticks = np.where(rng.random((T, n)) < 0.06, mode, STEP).astype(np.uint8)
    ticks[0] = NEXT_STEP_RESET  # an explicit reset first
    return ticks


@pytest.mark.parametrize("mode", [NEXT_STEP_RESET, SAME_STEP_RESET])
def test_schedule_matches_the_numpy_law(mode):
    L = _lib()
    rng = np.random.default_rng(mode)
    spec, seed, T, n, off = make_spec(gap=(0, 6), duration=(1, 5)), 5, 300, 24, 1000
    ticks = _random_ticks(rng, T, n, mode)
    applied, reported, count, timer = push_schedule_np(spec, seed, off + np.arange(n), ticks)
    assert 0.15 < np.mean(np.any(applied != 0, axis=2)) < 0.8  # both pushed and unpushed ticks
    for i in range(n):
        f = np.empty((T, 3), dtype=np.float32)
        k, t = np.empty(T, dtype=np.uint32), np.empty(T, dtype=np.uint32)
        col = np.ascontiguousarray(ticks[:, i])
        L.hostsim_push_run(C.byref(spec), seed, off + i, T, _p(col, C.c_uint8), 0, 0, _p(f, C.c_float),
                           _p(k, C.c_uint32), _p(t, C.c_uint32))
        np.testing.assert_array_equal(f, applied[:, i])
        np.testing.assert_array_equal(k, count[:, i])
        np.testing.assert_array_equal(t, timer[:, i])
        # what get_push_forces reports from the state after each tick
        for s in range(T):
            r = np.empty(3, dtype=np.float32)
            L.hostsim_push_last_force(C.byref(spec), seed, off + i, int(k[s]), int(t[s]), _p(r, C.c_float))
            np.testing.assert_array_equal(r, reported[s, i])


def test_schedule_follows_the_semantics():
    """gap steps without a push after a reset, duration steps of one constant force, the next draw"""
    spec, seed, g = make_spec(gap=(0, 4), duration=(1, 3)), 9, 77
    T = 200
    ticks = np.zeros((T, 1), dtype=np.uint8)
    ticks[0] = NEXT_STEP_RESET
    applied, _, count, _ = push_schedule_np(spec, seed, g, ticks)
    s, k = 1, 1
    while s < T:
        gap, dur, f = push_draw_np(spec, seed, g, k)
        for _ in range(int(gap[0])):
            if s < T:
                assert not applied[s, 0].any(), s
                s += 1
        for _ in range(int(dur[0])):
            if s < T:
                np.testing.assert_array_equal(applied[s, 0], f[0])
                s += 1
        k += 1
    assert count[-1, 0] >= 2


def test_explicit_reset_restarts_the_selected_envs():
    spec, seed, off, n = make_spec(), 4, 10, 6
    count = np.array([0, 3, 3, 7, 0, 2], dtype=np.uint32)
    gap, dur, _ = push_draw_np(spec, seed, off + np.arange(n), count)
    timer = np.array([0, 1, 0, 0, 5, 0], dtype=np.uint32)
    timer[2] = gap[2] + dur[2]  # its push ran out at the last step
    mask = np.array([1, 1, 1, 0, 1, 1], dtype=np.uint8)
    c, t = count.copy(), timer.copy()
    _lib().hostsim_push_reset(C.byref(spec), seed, off, n, _p(mask, C.c_uint8), _p(c, C.c_uint32), _p(t, C.c_uint32))
    assert (c[0], c[1], c[2], c[3], c[5]) == (1, 4, 5, 7, 3)  # +2 where the push had run out, env 3 not reset
    assert c[4] == (2 if timer[4] >= gap[4] + dur[4] else 1)
    np.testing.assert_array_equal(t, [0, 0, 0, 0, 0, 0])
    _, _, c2, t2 = push_schedule_np(spec, seed, off + np.arange(n), np.full((1, n), NEXT_STEP_RESET), count, timer)
    np.testing.assert_array_equal(c2[0][mask == 1], c[mask == 1])


def test_spec_validation():
    L = _lib()
    assert L.hostsim_push_spec_valid(C.byref(make_spec()))
    assert L.hostsim_push_spec_valid(C.byref(make_spec(body=6, gap=(0, 0), duration=(2**30, 2**30))))
    bad = [make_spec(body=-1), make_spec(body=7), make_spec(gap=(5, 4)), make_spec(duration=(3, 2)),
           make_spec(duration=(0, 3)), make_spec(gap=(0, 2**30 + 1)), make_spec(duration=(1, 2**31)),
           make_spec(force=((0, 0, 1), (0, 0, 0))), make_spec(force=((0, 0, 0), (np.inf, 0, 0))),
           make_spec(force=((np.nan, 0, 0), (1, 0, 0)))]
    for s in bad:
        assert not L.hostsim_push_spec_valid(C.byref(s))


# ---- the dict form ------------------------------------------------------------------------------------------------------


def test_dict_form_and_rounding():
    model, dt = default_model(), 0.005
    s = push_randomization_spec({"link": "torso", "interval": (1.0, 2.0), "duration": (0.1, 0.2),
                                 "force": ((-50.0, -10.0, 0.0), (50.0, 10.0, 0.0))}, model, dt)
    assert (s.body, s.gap_low, s.gap_high, s.duration_low, s.duration_high) == (0, 200, 400, 20, 40)
    assert list(s.force_low) == [-50.0, -10.0, 0.0] and list(s.force_high) == [50.0, 10.0, 0.0]
    # nearest step, halves up; lumped links map to their body; scalar force bounds
    s = push_randomization_spec({"link": "left_wheel_tire", "interval": (0.0, 0.0124), "duration": (0.0025, 0.0176),
                                 "force": (-1.0, 1.0)}, model, dt)
    assert (s.body, s.gap_low, s.gap_high, s.duration_low, s.duration_high) == (3, 0, 2, 1, 4)
    assert list(s.force_low) == [-1.0] * 3 and list(s.force_high) == [1.0] * 3
    assert push_randomization_spec(None, model, dt) is None


_GOOD = {"link": "torso", "interval": (0.5, 1.0), "duration": (0.05, 0.1), "force": ((-5, -5, 0), (5, 5, 0))}


@pytest.mark.parametrize("change", [
    {"kick": 1.0},                                    # unknown key
    {"link": "tail"},                                 # unknown link
    {"link": ["torso", "imu"]},                       # not one link name
    {"interval": (1.0, 0.5)},                         # low > high
    {"interval": (-0.1, 0.5)},                        # negative time
    {"duration": (0.001, 0.1)},                       # rounds to 0 steps
    {"duration": (0.0, 0.0)},
    {"duration": (0.1, np.inf)},
    {"interval": (0.0, 1e8)},                         # more than PUSH_MAX_STEPS steps
    {"force": ((0, 0, 1), (0, 0, 0))},                # low > high
    {"force": ((0, 0, 0), (1e39, 0, 0))},             # not finite in fp32
    {"force": ((np.nan, 0, 0), (1, 0, 0))},
    {"force": ((0, 0), (1, 1))},                      # not one or three axes
    {"duration": 0.1},                                # not a pair
    None,                                             # a key missing
])
def test_bad_specs_are_rejected_before_the_device(change):
    from upkie_b200.envs import B200VectorEnv

    spec = dict(_GOOD, **change) if change is not None else {k: v for k, v in _GOOD.items() if k != "force"}
    with pytest.raises(UpkieException):
        push_randomization_spec(spec, default_model(), 0.005)
    with pytest.raises(UpkieException):
        B200VectorEnv(4, "servos", push_randomization=spec)  # no device here: rejected before it is needed
