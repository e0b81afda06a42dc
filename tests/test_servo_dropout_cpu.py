# SPDX-License-Identifier: Apache-2.0
"""Servo reply dropouts (upkie_b200_set_servo_dropout): the C struct against its mirror; the draws, the per-cycle loss
rule, the holds and the latched view, compiled for the CPU (tests/hostsim/servo_dropout.cpp) and held bit for bit to a
NumPy statement of the law in include/upkie_b200.h; the family the host picks with dropouts set; the spec's validation
on both sides. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import servo_dropout_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
SEED = 0x5EED

_LIB = None
fp, u32p = C.POINTER(C.c_float), C.POINTER(C.c_uint32)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "servo_dropout.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_dropout_"), "libhostsim_servo_dropout.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_servo_dropout_run.argtypes = [vp, C.c_int, fp, fp, C.c_uint32, fp, u32p, C.c_uint64, C.c_uint64,
                                                C.c_int, fp, fp, fp]
        L.hostsim_servo_dropout_lost.restype = C.c_uint32
        L.hostsim_servo_dropout_lost.argtypes = [C.c_uint32, C.c_float, C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32]
        L.hostsim_servo_dropout_reset.argtypes = [C.c_int, fp, C.POINTER(_abi.UpkieServoDropout), C.c_uint64,
                                                  C.c_uint64, u32p, fp, fp]
        L.hostsim_servo_dropout_spec_error.argtypes = [C.POINTER(_abi.UpkieServoDropout), C.c_int, C.c_int, C.c_int,
                                                       C.c_char_p, C.c_int]
        L.hostsim_step_family_servo_dropout.argtypes = [C.c_int] * 6 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def prob_np(low, high, seed, g, k):
    """p_i of draw k of the envs of global index g (include/upkie_b200.h): fp32, the product rounded on its own"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    hi = np.uint64(1 << 59) | (np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4))
    w = philox_np(g, hi, np.full(g.shape, seed, dtype=np.uint64))[0]
    lo, hi_ = np.float32(low), np.float32(high)
    return np.minimum(lo + (hi_ - lo) * u01(w), hi_)


def lost_np(mask, p, seed, g, tick, sub):
    """[len(g), 6] the servos whose reply is lost in substep `sub` of tick `tick` (arrays broadcast over envs)"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    tick = np.broadcast_to(np.asarray(tick, dtype=np.uint64), g.shape)
    p = np.broadcast_to(np.asarray(p, dtype=np.float32), g.shape)
    out = np.zeros(g.shape + (6,), dtype=bool)
    for b in range(2):
        hi = np.uint64((1 << 59) | (1 << 58)) | (tick << np.uint64(20)) | np.uint64((sub << 1) | b)
        w = philox_np(g, hi, np.full(g.shape, seed, dtype=np.uint64))
        for k in range(4):
            j = 4 * b + k
            if j < 6 and (mask >> j) & 1:
                out[:, j] = u01(w[k]) < p
    return out


def ages_np(mask, prob, tick0, env_offset, nb, nticks):
    """[nticks * nb, n, 6] each servo's age at the end of every substep: 0 when its reply of that cycle arrived, k when
    its last one arrived k cycles earlier; an age reaching before the run points at the state the run starts from"""
    n = len(prob)
    g = env_offset + np.arange(n, dtype=np.uint64)
    ages = np.zeros((nticks * nb, n, 6), dtype=np.int64)
    age = np.full((n, 6), 10 ** 6, dtype=np.int64)  # the held rows start as the initial state (age: before the run)
    for t in range(nticks):
        for s in range(nb):
            lost = lost_np(mask, prob, SEED, g, tick0 + 1 + t, s)
            age = np.where(lost, age + 1, 0)
            ages[t * nb + s] = age
    return ages


class _Sim:
    def __init__(self, nb):
        self._m = default_model().to_struct()
        self._c = _abi.default_sim_config()
        self._c.nb_substeps = nb
        self.h = _lib().hostsim_create(C.byref(self._m), C.byref(self._c))
        assert self.h

    def __del__(self):
        try:
            _lib().hostsim_destroy(self.h)
        except Exception:
            pass


def _run(nb, n, mask, prob, nticks, seed=0, env_offset=3):
    rng = np.random.default_rng(seed)
    sim = _Sim(nb)
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    state[:, 2] = 0.58
    state[:, 3] = 1.0
    state[:, _abi.ST_Q:_abi.ST_Q + 6] = rng.normal(0.0, 0.3, size=(n, 6))
    state[:, _abi.ST_QD:_abi.ST_QD + 6] = rng.normal(0.0, 1.0, size=(n, 6))
    state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6] = rng.normal(0.0, 1.0, size=(n, 6))
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, 0] = rng.normal(0.0, 0.5, size=(n, 6))
    a[:, :, 1] = rng.normal(0.0, 1.0, size=(n, 6))
    a[:, :, 3] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 4] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 5] = rng.uniform(0.5, 16.0, size=(n, 6))
    cmd = np.ascontiguousarray(a.reshape(n, 36))
    init = np.stack([state[:, _abi.ST_Q:_abi.ST_Q + 6], state[:, _abi.ST_QD:_abi.ST_QD + 6],
                     state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6]], axis=-1).reshape(n, 18)
    held = np.ascontiguousarray(init.T)  # [18][n]: the state the run starts from latched
    prob = np.ascontiguousarray(prob, dtype=np.float32)
    tick0 = rng.integers(0, 1000, n).astype(np.uint32)
    truth = np.zeros((nticks * nb, n, 18), dtype=np.float32)
    seen = np.zeros_like(truth)
    _lib().hostsim_servo_dropout_run(sim.h, n, _p(state), _p(cmd), mask, _p(prob), _p(tick0, u32p), SEED, env_offset,
                                     nticks, _p(held), _p(truth), _p(seen))
    return init, tick0, truth, seen, held


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieServoDropout \{(.*?)\} UpkieServoDropout;", header, re.S).group(1)
    names = re.findall(r"\b(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _abi.UpkieServoDropout._fields_]
    assert C.sizeof(_abi.UpkieServoDropout) == 16


@pytest.mark.parametrize("nb", [1, 2, 5])
def test_latched_triples_are_the_state_at_the_numpy_age(nb):
    n, nticks, mask = 48, 3, 0b101101
    prob = np.linspace(0.0, 0.9, n).astype(np.float32)
    init, tick0, truth, seen, _ = _run(nb, n, mask, prob, nticks)
    ages = ages_np(mask, prob, tick0, 3, nb, nticks)
    assert ages.max() > 0 and (ages[:, :, [1, 4]] == 0).all()  # some replies lost, none of the unmasked servos'
    for k in range(nticks * nb):
        for j in range(6):
            a = ages[k, :, j]
            src = k - a
            expect = np.where((src >= 0)[:, None], truth[np.clip(src, 0, None), np.arange(n), 3 * j:3 * j + 3],
                              init[:, 3 * j:3 * j + 3])
            np.testing.assert_array_equal(seen[k, :, 3 * j:3 * j + 3], expect)


def test_no_loss_at_zero_probability_and_every_loss_at_one():
    n = 16
    _, _, truth, seen, _ = _run(5, n, 0x3F, np.zeros(n), 3)
    np.testing.assert_array_equal(seen, truth)
    init, _, truth, seen, held = _run(5, n, 0x3F, np.ones(n), 3)
    np.testing.assert_array_equal(seen, np.broadcast_to(init, seen.shape))  # the latched values until the next reset
    np.testing.assert_array_equal(held.T, init)
    assert not np.array_equal(truth[-1], init)


def test_loss_draws_match_the_numpy_law():
    g = np.arange(5, 45, dtype=np.uint64)
    for p in (0.0, 0.25, 1.0):
        for tick, sub in ((1, 0), (77, 4), (2 ** 31 + 5, 3)):
            lost = lost_np(0x3F, p, SEED, g, tick, sub)
            bits = [_lib().hostsim_servo_dropout_lost(0x3F, p, SEED, int(x), tick, sub) for x in g]
            np.testing.assert_array_equal(np.array([[(b >> j) & 1 for j in range(6)] for b in bits], bool), lost)
    # the mask selects servos, and a block of four unselected servos draws nothing
    assert all(_lib().hostsim_servo_dropout_lost(0b110000, 1.0, SEED, int(x), 9, 2) == 0b110000 for x in g)


def test_reset_draws_the_probability_and_latches_the_state():
    n = 64
    rng = np.random.default_rng(1)
    state = rng.normal(size=(n, _abi.STATE_DIM)).astype(np.float32)
    spec = _abi.UpkieServoDropout(0.05, 0.4, 0x3F, 0)
    count = np.full(n, 6, dtype=np.uint32)
    prob = np.zeros(n, dtype=np.float32)
    held = np.zeros((18, n), dtype=np.float32)
    _lib().hostsim_servo_dropout_reset(n, _p(state), C.byref(spec), SEED, 100, _p(count, u32p), _p(prob), _p(held))
    assert (count == 7).all()
    np.testing.assert_array_equal(prob, prob_np(0.05, 0.4, SEED, 100 + np.arange(n), 7))
    assert prob.min() >= np.float32(0.05) and prob.max() <= np.float32(0.4)
    for j in range(6):
        for k, col in enumerate((_abi.ST_Q, _abi.ST_QD, _abi.ST_TORQUE)):
            np.testing.assert_array_equal(held[3 * j + k], state[:, col + j])
    # sharding: the draw is keyed on the global env index
    np.testing.assert_array_equal(prob_np(0.05, 0.4, SEED, 100 + np.arange(32, 64), 7), prob[32:])


def _why(spec, limits=1, spine=0, body=0):
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_servo_dropout_spec_error(C.byref(spec), limits, spine, body, buf, 256)
    return buf.value.decode() if r else None


def test_spec_rejections():
    ok = _abi.UpkieServoDropout(0.0, 0.1, 0x3F, 0)
    assert _why(ok) is None
    assert _why(_abi.UpkieServoDropout(1.0, 1.0, 1, 0)) is None
    for lo, hi in ((-0.1, 0.2), (0.3, 0.2), (0.0, 1.5), (float("nan"), 0.1), (0.0, float("nan"))):
        assert _why(_abi.UpkieServoDropout(lo, hi, 0x3F, 0)) == "set_servo_dropout: 0 <= prob_low <= prob_high <= 1 required"
    for mask in (0, 0x40, 0x7F):
        assert "joint_mask" in _why(_abi.UpkieServoDropout(0.0, 0.1, mask, 0))
    assert "joint_limits" in _why(ok, limits=0)
    assert "spine_mode" in _why(ok, spine=1)
    assert "body_contacts" in _why(ok, body=1)


def _family(limits=1, spine=0, body=0, obs_delay=0, mode=0, transport=0):
    buf = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_servo_dropout(limits, spine, body, obs_delay, mode, transport, buf, 256)
    return f, buf.value.decode()


def test_family_choice():
    for mode in range(3):
        for transport in (0, 1):
            assert _family(mode=mode, transport=transport)[0] == FAM_SENSE
            assert _family(mode=mode, transport=transport, obs_delay=1)[0] == FAM_SENSE
    f, why = _family(transport=2)
    assert f == -1 and why == "servo dropouts have no in-kernel rollout transport (use upkie_b200_step with compact rows)"
    assert _family(spine=1) == (-1, "servo dropouts: spine_mode reports the spine's own servo replies")
    assert _family(limits=0) == (-1, "servo dropouts need joint_limits != 0")
    assert _family(body=1) == (-1, "servo dropouts have no body-contact kernels")


def test_python_spec_validation():
    s = servo_dropout_spec(0.1)
    assert (s.prob_low, s.prob_high, s.joint_mask) == (np.float32(0.1), np.float32(0.1), 0x3F)
    s = servo_dropout_spec((0.0, 0.2), ["left_wheel", "right_wheel"])
    assert s.joint_mask == (1 << 2) | (1 << 5)
    assert servo_dropout_spec(None) is None
    for bad in ((0.3, 0.2), -0.1, 1.5, (0.0, float("nan"))):
        with pytest.raises(UpkieException, match="servo_dropout"):
            servo_dropout_spec(bad)
    with pytest.raises(UpkieException, match="unknown joint"):
        servo_dropout_spec(0.1, ["left_elbow"])
    with pytest.raises(UpkieException, match="at least one"):
        servo_dropout_spec(0.1, [])
    for kw in ({"spine_mode": True}, {"joint_limits": 0}, {"body_contacts": True}):
        with pytest.raises(UpkieException, match="servo_dropout"):
            servo_dropout_spec(0.1, **kw)
