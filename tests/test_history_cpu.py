# SPDX-License-Identifier: Apache-2.0
"""Spine-rate observation history (upkie_b200_set_history): the C struct against its mirror; the history's column
arithmetic, ring order, reset fill and delayed window, compiled for the CPU (tests/hostsim/history.cpp) and held bit for
bit to the full spine observation of the state after each substep; the family the host picks with a history set; the
spec's validation on both sides and the key parser of the vector envs. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import history_spec, history_to_dict, spine_row_to_dict
from upkie_b200.model import default_model

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10

_LIB = None
fp, u32p, u8p, ip = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_uint8), C.POINTER(C.c_int)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "history.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_history_"), "libhostsim_history.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_history_run.argtypes = [vp, C.c_int, fp, fp, C.c_int, ip, C.c_int, C.c_int, C.c_int, fp, u32p, fp]
        L.hostsim_history_fill.argtypes = [vp, C.c_int, fp, C.c_int, ip, C.c_int, C.c_int, fp, u8p]
        L.hostsim_history_read.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, fp, u32p, u32p, fp]
        L.hostsim_history_spec_error.argtypes = [C.POINTER(_abi.UpkieHistory), C.c_int, C.c_int, C.c_int, C.c_char_p,
                                                 C.c_int]
        L.hostsim_step_family_history.argtypes = [C.c_int] * 7 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


class _Sim:
    def __init__(self, nb, n):
        self.n, self.nb = n, nb
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


def _start_state(n, rng):
    st = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    st[:, 2] = 0.58
    st[:, 3] = 1.0
    st[:, _abi.ST_Q:_abi.ST_Q + 6] = rng.normal(0.0, 0.3, size=(n, 6)).astype(np.float32)
    st[:, _abi.ST_ANGVEL:_abi.ST_ANGVEL + 3] = rng.normal(0.0, 0.5, size=(n, 3)).astype(np.float32)
    st[:, _abi.ST_LINVEL:_abi.ST_LINVEL + 3] = rng.normal(0.0, 0.2, size=(n, 3)).astype(np.float32)
    return st


def _servo_actions(n, rng):
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, 0] = rng.normal(0.0, 0.5, size=(n, 6))
    a[:, :, 1] = rng.normal(0.0, 1.0, size=(n, 6))
    a[:, :, 3] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 4] = rng.uniform(0.0, 1.5, size=(n, 6))
    a[:, :, 5] = rng.uniform(0.5, 16.0, size=(n, 6))
    return np.ascontiguousarray(a.reshape(n, 36))


# every column of the spine observation but the servo constants (temperature, voltage), 16 at a time
_MEASURED = [c for c in range(_abi.SPINE_DIM)
             if not (_abi.SP_SERVO <= c < _abi.SP_ODOM_POS and (c - _abi.SP_SERVO) % 5 >= 3)]
_GROUPS = [_MEASURED[k:k + 16] for k in range(0, len(_MEASURED), 16)]


def _run(nb, n, cols, size, ticks, nticks, seed=0):
    rng = np.random.default_rng(seed)
    sim = _Sim(nb, n)
    state = _start_state(n, rng)
    cmd = _servo_actions(n, rng)
    ring = np.zeros((ticks, len(cols), n), dtype=np.float32)
    head = np.zeros(n, dtype=np.uint32)
    spine = np.zeros((nticks * nb, n, _abi.SPINE_DIM), dtype=np.float32)
    c = np.asarray(cols, dtype=np.int32)
    _lib().hostsim_history_fill(sim.h, n, _p(state), len(cols), _p(c, ip), size, ticks, _p(ring), None)
    _lib().hostsim_history_run(sim.h, n, _p(state), _p(cmd), len(cols), _p(c, ip), size, ticks, nticks, _p(ring),
                               _p(head, u32p), _p(spine))
    return sim, state, ring, head, spine


def _read(ring, head, size, d):
    ticks, count, n = ring.shape
    out = np.zeros((n, size, count), dtype=np.float32)
    dd = np.ascontiguousarray(np.broadcast_to(np.asarray(d, dtype=np.uint32), (n,)))
    _lib().hostsim_history_read(n, count, size, ticks, _p(np.ascontiguousarray(ring)), _p(head, u32p), _p(dd, u32p),
                                _p(out))
    return out


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieHistory \{(.*?)\} UpkieHistory;", header, re.S).group(1)
    names = re.findall(r"(\w+)(?:\[\w+\])?\s*;", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f for f, _ in _abi.UpkieHistory._fields_]
    assert C.sizeof(_abi.UpkieHistory) == 8 + 4 * 16
    assert int(re.search(r"#define UPKIE_MAX_HISTORY (\d+)", header).group(1)) == _abi.MAX_HISTORY == 64
    assert int(re.search(r"#define UPKIE_MAX_HISTORY_CHANNELS (\d+)", header).group(1)) == _abi.MAX_HISTORY_CHANNELS
    for fn in ("upkie_b200_set_history", "upkie_b200_get_history", "upkie_b200_history_entries",
               "upkie_b200_get_history_state", "upkie_b200_set_history_state"):
        assert re.search(rf"\bint {fn}\(", header)
    assert "HistoryObserver.h" in header


@pytest.mark.parametrize("group", range(len(_GROUPS)))
@pytest.mark.parametrize("nb", [1, 5])
def test_ring_order_across_three_ticks_against_the_spine_observation(nb, group):
    """After 3 ticks, entry k is the spine observation of the state k substeps before the end, bit for bit, the IMU
    accelerations differentiated over one substep; entries cross the tick boundaries."""
    cols = _GROUPS[group]
    n, nticks = 6, 3
    size = 3 * nb
    ticks = size + nb
    _, _, ring, head, spine = _run(nb, n, cols, size, ticks, nticks)
    hist = _read(ring, head, size, 0)
    for k in range(size):
        ref = spine[nticks * nb - 1 - k][:, cols]
        np.testing.assert_array_equal(hist[:, k, :], ref, err_msg=f"entry {k}")


def test_entries_of_the_previous_tick_move_back_by_nb():
    nb, n, size = 5, 4, 10
    cols = [_abi.SP_PITCH, _abi.SP_IMU_ANGVEL, _abi.SP_IMU_LINACC + 2, _abi.SP_SERVO + 2 * 5 + 1]
    _, _, ring2, head2, _ = _run(nb, n, cols, size, size + nb, 2)
    _, _, ring3, head3, _ = _run(nb, n, cols, size, size + nb, 3)
    h2, h3 = _read(ring2, head2, size, 0), _read(ring3, head3, size, 0)
    np.testing.assert_array_equal(h3[:, nb:2 * nb], h2[:, 0:nb])


@pytest.mark.parametrize("d", [0, 1, 3, 5, 7, 10])
def test_delayed_window(d):
    """Under an observation delay of d substeps, entry k is the state d + k substeps before the end of the tick."""
    nb, n, size, nticks = 5, 3, 4, 3
    ticks = size + 2 * nb  # an observation delay of two ticks
    cols = [_abi.SP_BASE_ANGVEL + 1, _abi.SP_ODOM_VEL, _abi.SP_IMU_RAWACC]
    _, _, ring, head, spine = _run(nb, n, cols, size, ticks, nticks)
    hist = _read(ring, head, size, d)
    for k in range(size):
        np.testing.assert_array_equal(hist[:, k, :], spine[nticks * nb - 1 - d - k][:, cols])


def test_reset_fill_takes_the_masked_envs_only():
    nb, n, size = 5, 6, 7
    ticks = size + nb
    cols = [_abi.SP_PITCH, _abi.SP_IMU_LINACC, _abi.SP_SERVO + 1, _abi.SP_CONTACT]
    sim, state, ring, head, _ = _run(nb, n, cols, size, ticks, 2)
    before = _read(ring, head, size, 0)
    mask = np.array([1, 0, 0, 1, 0, 1], dtype=np.uint8)
    c = np.asarray(cols, dtype=np.int32)
    _lib().hostsim_history_fill(sim.h, n, _p(state), len(cols), _p(c, ip), size, ticks, _p(ring), _p(mask, u8p))
    after = _read(ring, head, size, 0)
    for i in range(n):
        if mask[i]:
            # every entry: the observation columns of the state, its own IMU acceleration
            assert (after[i] == after[i, :1]).all()
            assert np.isclose(after[i, 0, 0], np.arcsin(np.clip(2 * (state[i, 3] * state[i, 5] - state[i, 6] * state[i, 4]),
                                                                -1, 1)), atol=1e-6)
        else:
            np.testing.assert_array_equal(after[i], before[i])


def test_family_choice_and_rejections():
    L = _lib()
    why = C.create_string_buffer(256)
    for mode in (0, 1, 2):
        for transport in (0, 1):
            for od in (0, 1):
                for ad in (0, 1):
                    assert L.hostsim_step_family_history(3, 0, 0, od, ad, mode, transport, why, 256) == FAM_SENSE
    assert L.hostsim_step_family_history(3, 0, 0, 0, 0, 0, 2, why, 256) == -1
    assert b"history" in why.value and b"in-kernel" in why.value
    for args, word in (((0, 0, 0), b"joint_limits"), ((3, 0, 1), b"body-contact"), ((3, 1, 0), b"spine_mode")):
        assert L.hostsim_step_family_history(*args, 0, 0, 0, 0, why, 256) == -1
        assert b"history" in why.value and word in why.value


def test_spec_validation():
    L = _lib()
    why = C.create_string_buffer(256)

    def spec(size, cols):
        s = _abi.UpkieHistory(size, len(cols))
        for k, c in enumerate(cols):
            s.columns[k] = c
        return s

    assert L.hostsim_history_spec_error(spec(5, [6]), 3, 0, 0, why, 256) == 0
    assert L.hostsim_history_spec_error(spec(64, list(range(16))), 3, 0, 0, why, 256) == 0
    for s, word in ((spec(0, [6]), b"size"), (spec(65, [6]), b"size"), (spec(5, []), b"count"),
                    (spec(5, [-1]), b"column"), (spec(5, [62]), b"column")):
        assert L.hostsim_history_spec_error(s, 3, 0, 0, why, 256) == 1 and word in why.value
    s17 = _abi.UpkieHistory(5, 17)
    assert L.hostsim_history_spec_error(s17, 3, 0, 0, why, 256) == 1 and b"count" in why.value
    for (jl, sm, bc), word in (((0, 0, 0), b"joint_limits"), ((3, 1, 0), b"spine_mode"), ((3, 0, 1), b"body_contacts")):
        assert L.hostsim_history_spec_error(spec(5, [6]), jl, sm, bc, why, 256) == 1 and word in why.value


def test_key_parser_maps_keys_to_spine_columns():
    cols, size, layout = history_spec([("imu", "angular_velocity"), "base_orientation/pitch",
                                       ("servo", "left_wheel", "velocity"), ("servo", "right_hip", "torque"),
                                       ("wheel_odometry", "position")], 40)
    assert size == 40
    assert cols == [20, 21, 22, 6, 30 + 2 * 5 + 1, 30 + 3 * 5 + 2, 60]
    # the same columns as spine_row_to_dict reads for those keys
    row = np.arange(_abi.SPINE_DIM, dtype=np.float32)
    d = spine_row_to_dict(row)
    assert d["imu"]["angular_velocity"] == [20.0, 21.0, 22.0]
    assert d["servo"]["left_wheel"]["velocity"] == 41.0 and d["servo"]["right_hip"]["torque"] == 47.0
    # every key of the dictionary that is a measurement maps to the columns the dictionary reads it from
    cols_all, _, layout_all = history_spec([("base_orientation", "rotation_base_to_world"), ("imu", "orientation"),
                                            ("floor_contact", "contact")], 1)
    assert cols_all == list(range(7, 16)) + list(range(16, 20)) + [29]
    h = np.tile(np.asarray(cols_all, dtype=np.float32), (2, 1))  # K = 2 entries holding their column numbers
    out = history_to_dict(layout_all, h)
    assert out["base_orientation"]["rotation_base_to_world"][0] == d["base_orientation"]["rotation_base_to_world"]
    assert out["imu"]["orientation"][1] == d["imu"]["orientation"]
    assert out["floor_contact"]["contact"] == [True, True]
    h2 = history_to_dict(layout, np.arange(2 * 7, dtype=np.float32).reshape(2, 7))
    assert h2["imu"]["angular_velocity"] == [[0.0, 1.0, 2.0], [7.0, 8.0, 9.0]]
    assert h2["base_orientation"]["pitch"] == [3.0, 10.0]


@pytest.mark.parametrize("keys, size, word", [
    ([("servo", "left_hip", "temperature")], 5, "constant"),
    ([("servo", "left_hip", "voltage")], 5, "constant"),
    ([("imu", "magnetometer")], 5, "unknown"),
    ([("servo", "left_elbow", "position")], 5, "unknown"),
    ([("base_orientation", "rotation_base_to_world"), ("imu", "orientation"), ("imu", "angular_velocity"),
      ("imu", "linear_acceleration")], 5, "16"),
    ([("imu", "angular_velocity")], 0, "history_size"),
    ([("imu", "angular_velocity")], 65, "history_size"),
])
def test_key_parser_rejections(keys, size, word):
    with pytest.raises(UpkieException, match=word):
        history_spec(keys, size)


def test_key_parser_rejects_configurations():
    for kw, word in ((dict(spine_mode=True), "spine_mode"), (dict(joint_limits=0), "joint_limits"),
                     (dict(body_contacts=True), "body_contacts")):
        with pytest.raises(UpkieException, match=word):
            history_spec([("imu", "angular_velocity")], 5, **kw)
    assert history_spec(None) is None
