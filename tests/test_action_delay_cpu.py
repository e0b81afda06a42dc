# SPDX-License-Identifier: Apache-2.0
"""Action-delay randomisation (upkie_b200_set_action_delay): the C struct against its mirror, the draw and the delayed
tick the kernels run, compiled for the CPU (tests/hostsim/action_delay.cpp), against a NumPy statement of the draw and
against the same substeps composed from the single substep of every tick; the families the host picks with a delay;
the spec's validation on both sides. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import action_delay_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")

MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM = 0, 1, 2
DEVICE, HOST_TILE, IN_KERNEL = 0, 1, 2
FAM_TABLE, FAM_PUSH, FAM_BODY_PUSH, FAM_DELAY, FAM_BODY_DELAY, FAM_SPINE, FAM_BODY = 5, 6, 7, 8, 9, 3, 4
TRAITS = ("extras", "limits", "table", "reset_rand", "spine", "body", "push", "delay")


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieActionDelay \{(.*?)\} UpkieActionDelay;", header, re.S).group(1)
    names = re.findall(r"(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f for f, _ in _abi.UpkieActionDelay._fields_]
    assert C.sizeof(_abi.UpkieActionDelay) == 8
    for fn in ("upkie_b200_set_action_delay", "upkie_b200_get_action_delay_state", "upkie_b200_set_action_delay_state"):
        assert re.search(rf"\bint {fn}\(", header)


# ---- NumPy statement of the draw ----------------------------------------------------------------------------------------


def action_delay_draw_np(low, high, seed, env_index, k):
    """Draw k of the envs of global index env_index (arrays broadcast): the delay in substeps (uint32), as
    include/upkie_b200.h states the law"""
    g = np.atleast_1d(np.asarray(env_index, dtype=np.uint64))
    k = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape)
    hi_word = np.uint64(1 << 61) | (k << np.uint64(4))
    w0 = philox_np(g, hi_word, np.full(g.shape, seed, dtype=np.uint64))[0]
    return (np.uint64(low) + (((w0 >> np.uint32(8)).astype(np.uint64) * np.uint64(high - low + 1)) >> np.uint64(24))
            ).astype(np.uint32)


# ---- the CPU build of the kernels' code --------------------------------------------------------------------------------

_LIB = None
fp, u32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "action_delay.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_delay_"), "libhostsim_delay.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        sp, vp = C.POINTER(_abi.UpkieActionDelay), C.c_void_p
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_action_delay_draw.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_uint32]
        L.hostsim_action_delay_draw.restype = C.c_uint32
        L.hostsim_action_delay_reset.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_int, u8p, u32p, u32p, fp, C.c_int]
        L.hostsim_action_delay_tick.argtypes = [vp, C.c_int, C.c_int, fp, fp, fp, u32p, C.c_int, C.c_uint32,
                                                C.c_uint64, u32p]
        L.hostsim_servo_substeps.argtypes = [vp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_int, C.c_uint32, C.c_uint64,
                                             C.c_int]
        L.hostsim_action_delay_stop_row.argtypes = [fp]
        L.hostsim_gyropod_command.argtypes = [vp, C.c_int, fp, fp, fp]
        L.hostsim_step_servos_noise.argtypes = [vp, C.c_int, fp, fp, C.c_uint32, C.c_uint64, fp]
        L.hostsim_step_gyropod.argtypes = [vp, C.c_int, fp, fp, C.c_int, fp, u8p]
        L.hostsim_action_delay_spec_error.argtypes = [sp, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_family_traits_delay.argtypes = [C.c_int, u8p]
        L.hostsim_step_family_delay.argtypes = [C.c_int] * 9 + [C.c_char_p, C.c_int]
        L.hostsim_step_family_delay.restype = C.c_int
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


def draw_c(low, high, seed, g, k):
    return _lib().hostsim_action_delay_draw(C.byref(_abi.UpkieActionDelay(low, high)), seed, g, k)


@pytest.mark.parametrize("nb", [1, 2, 5, 10])
def test_draw_matches_numpy_bit_for_bit(nb):
    rng = np.random.default_rng(nb)
    for low in range(nb + 1):
        for high in range(low, nb + 1):
            seeds = [0, 1, 2**40 + 7, 2**64 - 1]
            for seed in seeds:
                g = rng.integers(0, 2**40, size=16, dtype=np.uint64)
                k = rng.integers(0, 2**32, size=16, dtype=np.uint64)
                ref = action_delay_draw_np(low, high, seed, g, k)
                got = [draw_c(low, high, seed, int(gi), int(ki)) for gi, ki in zip(g, k)]
                assert list(ref) == got
                assert np.all((ref >= low) & (ref <= high))


@pytest.mark.parametrize("low, high", [(0, 5), (1, 3), (0, 1), (2, 2), (5, 5), (0, 10)])
def test_draw_hits_every_value_of_its_range(low, high):
    d = action_delay_draw_np(low, high, 11, np.arange(4096, dtype=np.uint64), 1)
    assert set(d.tolist()) == set(range(low, high + 1))
    if low == high:
        assert np.all(d == low)


def test_draw_depends_on_global_index_and_counter_only():
    # a shard [offset, offset + n) of a batch draws what the whole batch draws there
    whole = action_delay_draw_np(0, 5, 3, np.arange(64, dtype=np.uint64), 4)
    shard = action_delay_draw_np(0, 5, 3, np.arange(32, 64, dtype=np.uint64), 4)
    assert np.array_equal(whole[32:], shard)
    # the tag keeps draws apart from the pushes' (bit 62) at the same (g, k)
    g, k = np.arange(256, dtype=np.uint64), np.uint64(1)
    push_w0 = philox_np(g, np.uint64(1 << 62) | (k << np.uint64(4)), np.full(g.shape, 3, dtype=np.uint64))[0]
    delay_w0 = philox_np(g, np.uint64(1 << 61) | (k << np.uint64(4)), np.full(g.shape, 3, dtype=np.uint64))[0]
    assert not np.array_equal(push_w0, delay_w0)


def test_reset_draws_and_stops():
    n, stride = 40, 64
    spec = _abi.UpkieActionDelay(1, 4)
    count = np.arange(n, dtype=np.uint32) % 3
    delay = np.full(n, 99, dtype=np.uint32)
    command = np.full((36, stride), 7.0, dtype=np.float32)
    mask = (np.arange(n) % 2).astype(np.uint8)
    count0 = count.copy()
    _lib().hostsim_action_delay_reset(C.byref(spec), 5, 100, n, _p(mask, u8p), _p(count, u32p), _p(delay, u32p),
                                      _p(command), stride)
    m = mask.astype(bool)
    assert np.array_equal(count[m], count0[m] + 1) and np.array_equal(count[~m], count0[~m])
    ref = action_delay_draw_np(1, 4, 5, 100 + np.arange(n, dtype=np.uint64), count0.astype(np.uint64) + 1)
    assert np.array_equal(delay[m], ref[m]) and np.all(delay[~m] == 99)
    cols = command[:, :n].T.reshape(n, 6, 6)
    assert np.all(np.isnan(cols[m][:, :, 0])) and np.all(cols[m][:, :, 1:] == 0.0)
    assert np.all(cols[~m] == 7.0) and np.all(command[:, n:] == 7.0)


# ---- the delayed tick --------------------------------------------------------------------------------------------------


def _config(nb, noise):
    c = _abi.default_sim_config()
    c.nb_substeps = nb
    for j in range(6):
        c.joint_friction[j] = 0.05
        c.torque_control_noise[j] = 0.3 if noise else 0.0
    c.noise_seed = 17
    return c


class _Sim:
    def __init__(self, nb, noise, n):
        self.n, self.nb, self.noise = n, nb, noise
        self._m = default_model().to_struct()
        self._c = _config(nb, noise)
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h

    def __del__(self):
        try:
            _lib().hostsim_destroy(self.h)
        except Exception:
            pass


def _start_state(n, rng):
    st = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    st[:, 2] = 0.58
    st[:, 3] = 1.0
    st[:, _abi.ST_Q:_abi.ST_Q + 6] = rng.normal(0.0, 0.3, size=(n, 6)).astype(np.float32)
    return st


def _servo_actions(n, rng):
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, 0] = rng.normal(0.0, 0.5, size=(n, 6))
    a[:, :, 1] = rng.normal(0.0, 1.0, size=(n, 6))
    a[:, :, 2] = rng.normal(0.0, 0.5, size=(n, 6))
    a[:, :, 3] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 4] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 5] = rng.uniform(0.5, 16.0, size=(n, 6))
    return a.reshape(n, 36)


def _tick(sim, mode, state, prev, action, d, tick=3):
    delay = np.full(sim.n, d, dtype=np.uint32) if np.isscalar(d) else np.asarray(d, dtype=np.uint32)
    err = np.zeros(sim.n, dtype=np.uint32)
    _lib().hostsim_action_delay_tick(sim.h, sim.n, mode, _p(state), _p(prev), _p(np.ascontiguousarray(action)),
                                     _p(delay, u32p), int(sim.noise), tick, 9, _p(err, u32p))
    return err


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD])
def test_zero_delay_is_todays_tick(mode, noise):
    if mode == MODE_GYROPOD and noise:
        pytest.skip("the gyropod tick of the CPU build has no noise entry point")
    n, nb = 8, 5
    rng = np.random.default_rng(1)
    sim = _Sim(nb, noise, n)
    state = _start_state(n, rng)
    prev = _servo_actions(n, rng)
    ref_state = state.copy()
    if mode == MODE_SERVOS:
        action = _servo_actions(n, rng)
        obs = np.empty((n, 30), dtype=np.float32)
        _lib().hostsim_step_servos_noise(sim.h, n, _p(ref_state), _p(action.copy()), 3, 9, _p(obs))
    else:
        action = rng.normal(0.0, 0.5, size=(n, 2)).astype(np.float32)
        o6, term = np.empty((n, 6), dtype=np.float32), np.empty(n, dtype=np.uint8)
        _lib().hostsim_step_gyropod(sim.h, n, _p(ref_state), _p(action.copy()), 2, _p(o6), _p(term, u8p))
    _tick(sim, mode, state, prev, action, 0)
    assert state.tobytes() == ref_state.tobytes()


@pytest.mark.parametrize("noise", [False, True])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD])
@pytest.mark.parametrize("nb", [2, 5])
def test_every_delay_is_the_composed_substeps(nb, mode, noise):
    n = 6
    rng = np.random.default_rng(nb + 10 * mode)
    sim = _Sim(nb, noise, n)
    state0 = _start_state(n, rng)
    prev0 = _servo_actions(n, rng)
    action = _servo_actions(n, rng) if mode == MODE_SERVOS else rng.normal(0.0, 0.5, size=(n, 2)).astype(np.float32)
    # the wrapper's yaw integration (gyropod) is not part of the substeps
    keep = np.ones(_abi.STATE_DIM, dtype=bool)
    keep[[_abi.ST_YAW, _abi.ST_YAW_VEL]] = mode == MODE_SERVOS
    for d in range(nb + 1):
        state, prev = state0.copy(), prev0.copy()
        _tick(sim, mode, state, prev, action, d)
        cur = prev.copy()  # the tick leaves its own command, clamped, in the buffer
        ref = state0.copy()
        if mode == MODE_GYROPOD:
            scratch = np.empty_like(cur)
            _lib().hostsim_gyropod_command(sim.h, n, _p(ref), _p(action.copy()), _p(scratch))
            assert scratch.tobytes() == cur.tobytes()
        _lib().hostsim_servo_substeps(sim.h, n, _p(ref), _p(prev0.copy()), 0, d, int(noise), 3, 9, 0)
        _lib().hostsim_servo_substeps(sim.h, n, _p(ref), _p(cur), d, nb, int(noise), 3, 9, 1)
        assert state[:, keep].tobytes() == ref[:, keep].tobytes(), f"d = {d}"
        if d > 0:
            other = state0.copy()
            _lib().hostsim_servo_substeps(sim.h, n, _p(other), _p(cur), 0, nb, int(noise), 3, 9, 1)
            assert other[:, keep].tobytes() != state[:, keep].tobytes()


@pytest.mark.parametrize("noise", [False, True])
def test_stop_row_gives_zero_torque(noise):
    n, nb = 16, 5
    rng = np.random.default_rng(3)
    sim = _Sim(nb, noise, n)
    state = _start_state(n, rng)
    state[:, _abi.ST_QD:_abi.ST_QD + 6] = rng.normal(0.0, 2.0, size=(n, 6)).astype(np.float32)  # friction acts
    stop = np.empty(36, dtype=np.float32)
    _lib().hostsim_action_delay_stop_row(_p(stop))
    rows = np.tile(stop, (n, 1))
    assert np.all(np.isnan(rows.reshape(n, 6, 6)[:, :, 0])) and np.all(rows.reshape(n, 6, 6)[:, :, 1:] == 0.0)
    ref = state.copy()
    _lib().hostsim_servo_substeps(sim.h, n, _p(state), _p(rows), 0, 1, int(noise), 3, 9, 0)
    # the torque the substep applied is the state's torque record
    assert np.all(state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6] == 0.0)
    assert state.tobytes() != ref.tobytes()


# ---- the families --------------------------------------------------------------------------------------------------------


def traits(family):
    out = (C.c_uint8 * len(TRAITS))()
    _lib().hostsim_family_traits_delay(family, out)
    return {name for name, v in zip(TRAITS, out) if v}


def step_family(mode=MODE_SERVOS, transport=DEVICE, joint_limits=2, table=0, body_contacts=0, push=0, delay=0,
                spine_mode=0, max_episode_steps=0):
    why = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_delay(joint_limits, table, body_contacts, push, delay, spine_mode,
                                         max_episode_steps, mode, transport, why, len(why))
    return f, (why.value.decode() or None)


def test_delay_traits():
    base = {"extras", "limits", "table", "reset_rand", "push"}
    assert traits(FAM_DELAY) == base | {"delay"}
    assert traits(FAM_BODY_DELAY) == base | {"body", "delay"}
    assert traits(FAM_DELAY) - {"delay"} == traits(FAM_PUSH)
    assert traits(FAM_BODY_DELAY) - {"delay"} == traits(FAM_BODY_PUSH)
    for fam in range(8):
        assert "delay" not in traits(fam)


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM])
def test_delay_families(mode, transport):
    assert step_family(mode, transport, delay=1) == (FAM_DELAY, None)
    assert step_family(mode, transport, delay=1, table=1) == (FAM_DELAY, None)
    assert step_family(mode, transport, delay=1, push=1) == (FAM_DELAY, None)
    assert step_family(mode, transport, delay=1, table=1, push=1, max_episode_steps=9) == (FAM_DELAY, None)
    assert step_family(mode, transport, delay=1, body_contacts=1) == (FAM_BODY_DELAY, None)
    assert step_family(mode, transport, delay=1, body_contacts=1, push=1) == (FAM_BODY_DELAY, None)
    # without a delay the choice is the one before the feature
    assert step_family(mode, transport, push=1) == (FAM_PUSH, None)
    assert step_family(mode, transport, table=1) == (FAM_TABLE, None)
    assert step_family(mode, transport, body_contacts=1) == (FAM_BODY, None)


NO_PUSH = "push randomisation has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
NO_DELAY = "action delay has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
NO_TABLE = "the per-env parameter table has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
NO_LIMIT = ("max_episode_steps has no in-kernel rollout transport: it does not carry truncated (use upkie_b200_step "
            "with compact rows)")


def test_in_kernel_transport_rejects_a_delay_after_the_push_message():
    assert step_family(MODE_SERVOS, IN_KERNEL, delay=1) == (-1, NO_DELAY)
    assert step_family(MODE_SERVOS, IN_KERNEL, delay=1, push=1)[1] == NO_PUSH
    assert step_family(MODE_SERVOS, IN_KERNEL, delay=1, table=1)[1] == NO_TABLE
    assert step_family(MODE_SERVOS, IN_KERNEL, delay=1, max_episode_steps=1, body_contacts=1)[1] == NO_DELAY
    assert step_family(MODE_SERVOS, IN_KERNEL, max_episode_steps=1)[1] == NO_LIMIT


# ---- the spec ------------------------------------------------------------------------------------------------------------


def spec_error(low, high, nb=5, joint_limits=3, spine_mode=0):
    why = C.create_string_buffer(256)
    rc = _lib().hostsim_action_delay_spec_error(C.byref(_abi.UpkieActionDelay(low, high)), nb, joint_limits,
                                                spine_mode, why, len(why))
    return why.value.decode() if rc else None


def test_c_spec_rejections():
    assert spec_error(0, 0) is None and spec_error(0, 5) is None and spec_error(5, 5) is None
    assert "substeps_low > substeps_high" in spec_error(3, 2)
    assert "above nb_substeps" in spec_error(0, 6)
    assert "joint_limits" in spec_error(0, 1, joint_limits=0)
    assert "spine_mode" in spec_error(0, 1, spine_mode=1)


def test_action_delay_spec_rounding():
    dt = 1.0 / 200.0  # 5 substeps of 1 ms
    assert action_delay_spec(None, dt, 5) is None
    assert action_delay_spec(0.0, dt, 5) == (0, 0)
    assert action_delay_spec(0.002, dt, 5) == (2, 2)
    assert action_delay_spec(0.0024, dt, 5) == (2, 2)
    assert action_delay_spec(0.0025, dt, 5) == (3, 3)  # halves up
    assert action_delay_spec((0.001, 0.005), dt, 5) == (1, 5)
    assert action_delay_spec((0, 0.0052), dt, 5) == (0, 5)  # rounds to one tick
    assert action_delay_spec(np.float32(0.003), dt, 5) == (3, 3)
    assert action_delay_spec(0.01, 1.0 / 100.0, 10) == (10, 10)


@pytest.mark.parametrize("bad, kw, match", [
    (-0.001, {}, "0 <= low <= high"),
    ((0.003, 0.002), {}, "0 <= low <= high"),
    (float("nan"), {}, "finite"),
    ((0.0, float("inf")), {}, "finite"),
    (0.006, {}, "more than one tick"),
    ((0.0, 0.0056), {}, "more than one tick"),
    ("abc", {}, "expected"),
    ((1, 2, 3), {}, "pair"),
    (0.001, {"spine_mode": True}, "spine_mode"),
    (0.001, {"joint_limits": False}, "joint_limits"),
    (0.001, {"joint_limits": 0}, "joint_limits"),
])
def test_action_delay_spec_rejections(bad, kw, match):
    with pytest.raises(UpkieException, match=match):
        action_delay_spec(bad, 1.0 / 200.0, 5, **kw)
