# SPDX-License-Identifier: Apache-2.0
"""Observation-delay randomisation (upkie_b200_set_observation_delay): the C struct against its mirror, the draw and the
snapshots the kernels take, compiled for the CPU (tests/hostsim/observation_delay.cpp), against a NumPy statement of the
draw and against the same substeps run without a delay; the family the host picks with a spec set, for every feature
combination; the spec's validation on both sides. No GPU needed."""
import ctypes as C
import itertools
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi, build
from upkie_b200.envs import observation_delay_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")

MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM = 0, 1, 2
DEVICE, HOST_TILE, IN_KERNEL = 0, 1, 2
FAM_SENSE = 10
FEATURES = ("joint_limits", "ctrl_noise", "meas_noise", "ext", "table", "body_contacts", "push", "delay", "spine_mode",
            "max_episode_steps", "sense")
TRAITS = ("extras", "limits", "table", "reset_rand", "spine", "body", "push", "delay", "sense")


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieObservationDelay \{(.*?)\} UpkieObservationDelay;", header, re.S).group(1)
    names = re.findall(r"(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f for f, _ in _abi.UpkieObservationDelay._fields_]
    assert C.sizeof(_abi.UpkieObservationDelay) == 8
    for fn in ("upkie_b200_set_observation_delay", "upkie_b200_get_observation_delay_state",
               "upkie_b200_set_observation_delay_state"):
        assert re.search(rf"\bint {fn}\(", header)


# ---- NumPy statement of the draw ----------------------------------------------------------------------------------------


def observation_delay_draw_np(low, high, seed, env_index, k, tag_bit=60):
    """Draw k of the envs of global index env_index (arrays broadcast): the delay in substeps (uint32), as
    include/upkie_b200.h states the law"""
    g = np.atleast_1d(np.asarray(env_index, dtype=np.uint64))
    k = np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape)
    hi_word = np.uint64(1 << tag_bit) | (k << np.uint64(4))
    w0 = philox_np(g, hi_word, np.full(g.shape, seed, dtype=np.uint64))[0]
    return (np.uint64(low) + (((w0 >> np.uint32(8)).astype(np.uint64) * np.uint64(high - low + 1)) >> np.uint64(24))
            ).astype(np.uint32)


# ---- the CPU build of the kernels' code --------------------------------------------------------------------------------

_LIB = None
fp, u32p, u8p = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "observation_delay.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_sense_"), "libhostsim_sense.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        sp, vp = C.POINTER(_abi.UpkieObservationDelay), C.c_void_p
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_obs_delay_draw.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_uint32]
        L.hostsim_obs_delay_draw.restype = C.c_uint32
        L.hostsim_obs_delay_reset.argtypes = [sp, C.c_uint64, C.c_uint64, C.c_int, u8p, u32p, u32p]
        L.hostsim_obs_delay_tick.argtypes = [vp, C.c_int, fp, fp, fp, u32p, fp]
        L.hostsim_obs_substeps.argtypes = [vp, C.c_int, fp, fp, C.c_int, C.c_int, C.c_int]
        L.hostsim_imu_velocity.argtypes = [vp, C.c_int, fp, fp]
        L.hostsim_obs_delay_sensed_columns.argtypes = [u8p]
        L.hostsim_obs_delay_spec_error.argtypes = [sp, C.c_int, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_step_family_sense.argtypes = [C.c_int] * (len(FEATURES) + 2) + [C.c_char_p, C.c_int]
        L.hostsim_step_family_sense.restype = C.c_int
        L.hostsim_family_traits_sense.argtypes = [C.c_int, u8p]
        L.hostsim_step_instantiated_sense.argtypes = [C.c_int, C.c_int]
        L.hostsim_step_instantiated_sense.restype = C.c_int
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


def draw_c(low, high, seed, g, k):
    return _lib().hostsim_obs_delay_draw(C.byref(_abi.UpkieObservationDelay(low, high)), seed, g, k)


@pytest.mark.parametrize("nb", [1, 2, 5, 10])
def test_draw_matches_numpy_bit_for_bit(nb):
    rng = np.random.default_rng(nb)
    for low in range(nb + 1):
        for high in range(low, nb + 1):
            for seed in (0, 1, 2**40 + 7, 2**64 - 1):
                g = rng.integers(0, 2**40, size=16, dtype=np.uint64)
                k = rng.integers(0, 2**32, size=16, dtype=np.uint64)
                ref = observation_delay_draw_np(low, high, seed, g, k)
                got = [draw_c(low, high, seed, int(gi), int(ki)) for gi, ki in zip(g, k)]
                assert list(ref) == got
                assert np.all((ref >= low) & (ref <= high))


def test_draw_hits_every_value_and_stays_apart_from_the_action_delay():
    d = observation_delay_draw_np(0, 5, 11, np.arange(4096, dtype=np.uint64), 1)
    assert set(d.tolist()) == set(range(6))
    # a shard [offset, offset + n) of a batch draws what the whole batch draws there
    whole = observation_delay_draw_np(0, 5, 3, np.arange(64, dtype=np.uint64), 4)
    assert np.array_equal(whole[32:], observation_delay_draw_np(0, 5, 3, np.arange(32, 64, dtype=np.uint64), 4))
    # the tag (bit 60) keeps the draws apart from the action delay's (bit 61) at the same (g, k)
    act = observation_delay_draw_np(0, 5, 3, np.arange(64, dtype=np.uint64), 4, tag_bit=61)
    assert not np.array_equal(whole, act)


def test_reset_counts_and_draws():
    n = 8
    count = np.array([0, 3, 7, 0, 1, 2, 9, 4], dtype=np.uint32)
    delay = np.zeros(n, dtype=np.uint32)
    mask = np.array([1, 0, 1, 1, 0, 1, 1, 0], dtype=np.uint8)
    before = count.copy()
    _lib().hostsim_obs_delay_reset(C.byref(_abi.UpkieObservationDelay(1, 4)), 21, 100, n, _p(mask, u8p),
                                   _p(count, u32p), _p(delay, u32p))
    sel = mask.astype(bool)
    assert np.array_equal(count[sel], before[sel] + 1) and np.array_equal(count[~sel], before[~sel])
    ref = observation_delay_draw_np(1, 4, 21, 100 + np.arange(n, dtype=np.uint64), count)
    assert np.array_equal(delay[sel], ref[sel]) and np.all(delay[~sel] == 0)


def test_sensed_columns():
    out = np.zeros(_abi.STATE_DIM, dtype=np.uint8)
    _lib().hostsim_obs_delay_sensed_columns(_p(out, u8p))
    sensed = set(range(_abi.ST_LEG_TARGET)) | {_abi.ST_CONTACT} | set(range(_abi.ST_IMU_ACC, _abi.ST_IMU_ACC + 3))
    assert {k for k in range(_abi.STATE_DIM) if out[k]} == sensed


# ---- the snapshot law ------------------------------------------------------------------------------------------------


class _Sim:
    def __init__(self, nb, n):
        self.n, self.nb = n, nb
        self._m = default_model().to_struct()
        self._c = _abi.default_sim_config()
        self._c.nb_substeps = nb
        for j in range(6):
            self._c.joint_friction[j] = 0.05
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h
        self.dt = float(self._c.dt)

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
    st[:, _abi.ST_ANGVEL:_abi.ST_ANGVEL + 3] = rng.normal(0.0, 0.5, size=(n, 3)).astype(np.float32)
    return st


def _servo_actions(n, rng):
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, 0] = rng.normal(0.0, 0.5, size=(n, 6))
    a[:, :, 1] = rng.normal(0.0, 1.0, size=(n, 6))
    a[:, :, 3] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 4] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 5] = rng.uniform(0.5, 16.0, size=(n, 6))
    return np.ascontiguousarray(a.reshape(n, 36))


def _imu_velocity(sim, state):
    v = np.zeros((len(state), 3), dtype=np.float32)
    _lib().hostsim_imu_velocity(sim.h, len(state), _p(np.ascontiguousarray(state)), _p(v))
    return v


SENSED = [k for k in range(_abi.STATE_DIM)
          if k < _abi.ST_LEG_TARGET or k == _abi.ST_CONTACT or _abi.ST_IMU_ACC <= k < _abi.ST_IMU_ACC + 3]
OTHERS = [k for k in range(_abi.STATE_DIM) if k not in SENSED]
BODY = [k for k in SENSED if not (_abi.ST_PREV_IMU_VEL <= k < _abi.ST_PREV_IMU_VEL + 3)
        and not (_abi.ST_IMU_ACC <= k < _abi.ST_IMU_ACC + 3)]


@pytest.mark.parametrize("nb", [1, 3, 5])
def test_snapshot_law_for_every_delay(nb):
    n = 6
    rng = np.random.default_rng(nb)
    sim = _Sim(nb, n)
    start = _start_state(n, rng)
    # a first undelayed tick, so that the state holds torques, contacts and an IMU pair of its own
    warm = _servo_actions(n, rng)
    _lib().hostsim_obs_substeps(sim.h, n, _p(start), _p(warm), 0, nb, 1)
    action = _servo_actions(n, rng)
    for d in range(nb + 1):
        state = start.copy()
        sensed = start.copy()  # the previous snapshot: the state itself (as after a reset)
        obs = np.zeros((n, _abi.OBS_DIM), dtype=np.float32)
        delay = np.full(n, d, dtype=np.uint32)
        _lib().hostsim_obs_delay_tick(sim.h, n, _p(state), _p(sensed), _p(action), _p(delay, u32p), _p(obs))
        # the true state is the undelayed tick's, whatever d
        ref = start.copy()
        _lib().hostsim_obs_substeps(sim.h, n, _p(ref), _p(action), 0, nb, 1)
        assert np.array_equal(state.view(np.uint32), ref.view(np.uint32)), d
        # the sensed fields are the state after nb - d substeps; the others the true state's
        part = start.copy()
        _lib().hostsim_obs_substeps(sim.h, n, _p(part), _p(action), 0, nb - d, 0)
        assert np.array_equal(sensed[:, BODY], part[:, BODY]), d
        assert np.array_equal(sensed[:, OTHERS], state[:, OTHERS]), d
        # the IMU pair: the snapshot's IMU velocity, differentiated against the previous snapshot's over dt
        got_v = sensed[:, _abi.ST_PREV_IMU_VEL:_abi.ST_PREV_IMU_VEL + 3]
        np.testing.assert_allclose(got_v, _imu_velocity(sim, part), rtol=0, atol=1e-6)
        prev = start[:, _abi.ST_PREV_IMU_VEL:_abi.ST_PREV_IMU_VEL + 3]
        acc = sensed[:, _abi.ST_IMU_ACC:_abi.ST_IMU_ACC + 3]
        np.testing.assert_allclose(acc, (got_v - prev) / np.float32(sim.dt), rtol=1e-5, atol=1e-3)
        # the observation rows are built from the sensed state
        o = obs.reshape(n, 6, 5)
        assert np.array_equal(o[:, :, 0], sensed[:, _abi.ST_Q:_abi.ST_Q + 6])
        assert np.array_equal(o[:, :, 1], sensed[:, _abi.ST_QD:_abi.ST_QD + 6])
        assert np.array_equal(o[:, :, 2], sensed[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6])
        if d == 0:  # today's observation, bit for bit: the whole row is the true state
            assert np.array_equal(sensed.view(np.uint32), state.view(np.uint32))
        if d == nb:  # the state at the start of the tick
            assert np.array_equal(sensed[:, BODY], start[:, BODY])


def test_imu_pair_follows_consecutive_snapshots():
    nb, n = 5, 4
    rng = np.random.default_rng(3)
    sim = _Sim(nb, n)
    state = _start_state(n, rng)
    sensed = state.copy()
    obs = np.zeros((n, _abi.OBS_DIM), dtype=np.float32)
    delay = np.array([0, 2, 4, 5], dtype=np.uint32)
    prev_v = sensed[:, _abi.ST_PREV_IMU_VEL:_abi.ST_PREV_IMU_VEL + 3].copy()
    for _ in range(4):
        action = _servo_actions(n, rng)
        _lib().hostsim_obs_delay_tick(sim.h, n, _p(state), _p(sensed), _p(action), _p(delay, u32p), _p(obs))
        v = sensed[:, _abi.ST_PREV_IMU_VEL:_abi.ST_PREV_IMU_VEL + 3]
        acc = sensed[:, _abi.ST_IMU_ACC:_abi.ST_IMU_ACC + 3]
        np.testing.assert_allclose(acc, (v - prev_v) / np.float32(sim.dt), rtol=1e-6, atol=1e-4)
        prev_v = v.copy()


# ---- the family choice -------------------------------------------------------------------------------------------------


def step_family(mode=MODE_SERVOS, transport=DEVICE, **features):
    assert set(features) <= set(FEATURES)
    why = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_sense(*(features.get(k, 0) for k in FEATURES), mode, transport, why, len(why))
    return f, (why.value.decode() or None)


def test_sense_traits():
    out = (C.c_uint8 * len(TRAITS))()
    _lib().hostsim_family_traits_sense(FAM_SENSE, out)
    assert {t for t, v in zip(TRAITS, out) if v} == {"extras", "limits", "table", "reset_rand", "push", "delay",
                                                      "sense"}
    for fam in range(FAM_SENSE):
        _lib().hostsim_family_traits_sense(fam, out)
        assert not out[TRAITS.index("sense")]
    assert all(_lib().hostsim_step_instantiated_sense(t, FAM_SENSE) for t in (DEVICE, HOST_TILE))
    assert not _lib().hostsim_step_instantiated_sense(IN_KERNEL, FAM_SENSE)
    units = [u for u in build.UNITS if isinstance(u, build.StepUnit) and FAM_SENSE in u.families]
    assert sorted(u.tile for u in units) == [DEVICE, HOST_TILE] and all(u.body == 0 for u in units)


@pytest.mark.parametrize("transport", [DEVICE, HOST_TILE, IN_KERNEL])
@pytest.mark.parametrize("mode", [MODE_SERVOS, MODE_GYROPOD, MODE_PENDULUM])
def test_every_feature_combination(mode, transport):
    # every combination of the features step_family reads, the observation delay included: a rejection, or an
    # instantiated pair; without the delay the choice is the one before the feature; with it, FAM_SENSE
    for values in itertools.product((0, 1), repeat=len(FEATURES)):
        kw = dict(zip(FEATURES, values))
        family, why = step_family(mode, transport, **kw)
        if family < 0:
            assert why, kw
        else:
            assert why is None and _lib().hostsim_step_instantiated_sense(transport, family), (kw, family)
        if not kw["sense"]:
            continue
        if transport == IN_KERNEL:
            assert family < 0
        elif kw["spine_mode"] or not kw["joint_limits"] or kw["body_contacts"]:
            assert family < 0, kw
        else:
            assert (family, why) == (FAM_SENSE, None), kw


def test_rejection_messages():
    no_sense = "observation delay has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
    no_delay = "action delay has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
    assert step_family(MODE_SERVOS, IN_KERNEL, joint_limits=2, sense=1) == (-1, no_sense)
    # right after the action delay's message
    assert step_family(MODE_SERVOS, IN_KERNEL, joint_limits=2, sense=1, delay=1)[1] == no_delay
    assert step_family(MODE_SERVOS, IN_KERNEL, joint_limits=2, sense=1, max_episode_steps=1)[1] == no_sense
    assert step_family(MODE_SERVOS, DEVICE, sense=1)[1] == "observation delay needs joint_limits != 0"
    assert step_family(MODE_SERVOS, DEVICE, joint_limits=2, sense=1, body_contacts=1)[1] == \
        "observation delay has no body-contact kernels"
    assert step_family(MODE_SERVOS, DEVICE, joint_limits=2, sense=1, spine_mode=1)[1] == \
        "observation delay: spine_mode models the spine's own lag"
    for kw in ({}, {"delay": 1}, {"push": 1}, {"table": 1, "delay": 1, "push": 1, "max_episode_steps": 5}):
        assert step_family(MODE_GYROPOD, HOST_TILE, joint_limits=3, sense=1, **kw) == (FAM_SENSE, None)


# ---- the spec ----------------------------------------------------------------------------------------------------------


def spec_error(low, high, nb=5, joint_limits=2, spine_mode=0, body_contacts=0):
    why = C.create_string_buffer(256)
    r = _lib().hostsim_obs_delay_spec_error(C.byref(_abi.UpkieObservationDelay(low, high)), nb, joint_limits,
                                            spine_mode, body_contacts, why, len(why))
    return why.value.decode() if r else None


def test_spec_validation_on_the_c_side():
    assert spec_error(0, 5) is None and spec_error(2, 2) is None and spec_error(0, 0) is None
    assert "substeps_low > substeps_high" in spec_error(3, 2)
    assert "above nb_substeps" in spec_error(0, 6)
    assert "joint_limits" in spec_error(0, 1, joint_limits=0)
    assert "spine_mode" in spec_error(0, 1, spine_mode=1)
    assert "body_contacts" in spec_error(0, 1, body_contacts=1)


def test_spec_rounding_and_rejections():
    dt, nb = 0.005, 5  # substeps of 1 ms
    assert observation_delay_spec(None, dt, nb) is None
    assert observation_delay_spec(0.0, dt, nb) == (0, 0)
    assert observation_delay_spec(0.002, dt, nb) == (2, 2)
    assert observation_delay_spec((0.0, 0.005), dt, nb) == (0, 5)
    assert observation_delay_spec((0.0014, 0.0026), dt, nb) == (1, 3)
    assert observation_delay_spec(0.0015, dt, nb) == (2, 2)  # halves up
    assert observation_delay_spec(np.float32(0.001), dt, nb) == (1, 1)
    for bad in ((0.003, 0.001), -0.001, float("nan"), (0.0, float("inf")), "x", (1, 2, 3), 0.0056):
        with pytest.raises(UpkieException):
            observation_delay_spec(bad, dt, nb)
    with pytest.raises(UpkieException, match="spine_mode"):
        observation_delay_spec(0.001, dt, nb, spine_mode=True)
    with pytest.raises(UpkieException, match="joint_limits"):
        observation_delay_spec(0.001, dt, nb, joint_limits=0)
    with pytest.raises(UpkieException, match="body_contacts"):
        observation_delay_spec(0.001, dt, nb, body_contacts=1)
