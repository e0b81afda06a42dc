# SPDX-License-Identifier: Apache-2.0
"""IMU mounting misalignment (upkie_b200_set_imu_misalignment): the C struct against its mirror; the draw law and the
reset compiled for the CPU (tests/hostsim/imu_misalignment.cpp) against a NumPy statement of include/upkie_b200.h; the
spine and gyropod observations read through the misalignment against an fp64 restatement that tilts the IMU frame
itself (not the base quaternion); the family the host picks with a misalignment set; the spec's validation on both
sides. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import imu_misalignment_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
SEED = 0x7117
RBI = np.diag([-1.0, 1.0, -1.0])  # rotation_base_to_imu of the default model

_LIB = None
fp, u32p, ip = C.POINTER(C.c_float), C.POINTER(C.c_uint32), C.POINTER(C.c_int)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "imu_misalignment.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_tilt_"), "libhostsim_imu_misalignment.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        spec_p = C.POINTER(_abi.UpkieImuMisalignment)
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_imu_misalign_draw.argtypes = [spec_p, C.c_uint64, C.c_uint64, C.c_uint32, fp]
        L.hostsim_imu_misalign_reset.argtypes = [C.c_int, spec_p, C.c_uint64, C.c_uint64, u32p, fp]
        L.hostsim_imu_misalign_obs.argtypes = [vp, C.c_int, fp, fp, fp, fp, ip]
        L.hostsim_imu_misalign_spec_error.argtypes = [spec_p, C.c_int, C.c_int, C.c_int, C.c_char_p, C.c_int]
        L.hostsim_step_family_imu_misalign.argtypes = [C.c_int] * 6 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a, t=fp):
    return a.ctypes.data_as(t)


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def angles_np(spec, seed, g, k):
    """[len(g), 3] roll, pitch and yaw of draw k of the envs of global index g (include/upkie_b200.h): fp32, the
    product rounded on its own, clamped to high"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    hi = np.uint64(1 << 57) | (np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4))
    w = philox_np(g, hi, np.full(g.shape, seed, dtype=np.uint64))
    out = np.zeros(g.shape + (3,), dtype=np.float32)
    for a, (lo, high) in enumerate(((spec.roll_low, spec.roll_high), (spec.pitch_low, spec.pitch_high),
                                    (spec.yaw_low, spec.yaw_high))):
        lo, high = np.float32(lo), np.float32(high)
        out[:, a] = np.minimum(lo + (high - lo) * u01(w[a]), high)
    return out


def quat_np(angles):
    """[n, 4] the unit quaternions (w, x, y, z) of Rz(yaw) Ry(pitch) Rx(roll), fp64"""
    a = np.asarray(angles, dtype=np.float64)
    return Rotation.from_euler("ZYX", a[:, ::-1]).as_quat(scalar_first=True)


def observe_np(state, e, rbi=RBI):
    """fp64 restatement: the IMU is mounted rotated by E (e, wxyz) in the base frame, so its true frame-to-world rotation
    is R E Rbi^T; it reports orientation, rate and accelerations in that frame, and the observers assume the nominal
    mounting (BaseOrientation.h), deriving the base orientation as (imu to world) Rbi. Returns a dict of [n, ...]."""
    s = np.asarray(state, dtype=np.float64)
    R = Rotation.from_quat(s[:, _abi.ST_QUAT:_abi.ST_QUAT + 4], scalar_first=True).as_matrix()
    E = Rotation.from_quat(np.asarray(e, dtype=np.float64), scalar_first=True).as_matrix()
    riw = R @ E @ rbi.T  # the true IMU frame to world
    omega = s[:, _abi.ST_ANGVEL:_abi.ST_ANGVEL + 3]
    acc = s[:, _abi.ST_IMU_ACC:_abi.ST_IMU_ACC + 3]
    gyro = np.einsum("nji,nj->ni", riw, omega)
    lin = np.einsum("nji,nj->ni", riw, acc)
    raw = np.einsum("nji,nj->ni", riw, acc + np.array([0.0, 0.0, 9.81]))
    rb = riw @ rbi  # the base orientation the observers derive
    ars = np.diag([1.0, -1.0, -1.0]) @ riw
    q_imu = Rotation.from_matrix(ars).as_quat(scalar_first=True)
    base_w = np.einsum("ij,nj->ni", rbi.T, gyro)  # rotation_imu_to_base * angular_velocity_imu_in_imu
    return {"rot": rb, "pitch": -np.arcsin(np.clip(rb[:, 2, 0], -1.0, 1.0)), "base_angvel": base_w, "imu_quat": q_imu,
            "imu_angvel": gyro, "imu_linacc": lin, "imu_rawacc": raw}


def check_spine(spine, ref, atol=2e-5, label=""):
    """the orientation-derived columns of spine rows [n, SPINE_DIM] against observe_np (fp32 tolerance)"""
    np.testing.assert_allclose(spine[:, _abi.SP_PITCH], ref["pitch"], atol=atol, err_msg=label)
    np.testing.assert_allclose(spine[:, _abi.SP_ROT:_abi.SP_ROT + 9], ref["rot"].reshape(-1, 9), atol=atol,
                               err_msg=label)
    np.testing.assert_allclose(spine[:, _abi.SP_BASE_ANGVEL:_abi.SP_BASE_ANGVEL + 3], ref["base_angvel"],
                               atol=atol * 10, rtol=1e-5, err_msg=label)
    q = spine[:, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4].astype(np.float64)
    sign = np.where(np.sum(q * ref["imu_quat"], axis=1) < 0, -1.0, 1.0)[:, None]  # q and -q: one rotation
    np.testing.assert_allclose(q * sign, ref["imu_quat"], atol=atol, err_msg=label)
    for key, col in (("imu_angvel", _abi.SP_IMU_ANGVEL), ("imu_linacc", _abi.SP_IMU_LINACC),
                     ("imu_rawacc", _abi.SP_IMU_RAWACC)):
        np.testing.assert_allclose(spine[:, col:col + 3], ref[key], atol=atol * 10, rtol=1e-5, err_msg=label + key)


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


def random_states(n, rng):
    state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
    state[:, _abi.ST_POS:_abi.ST_POS + 3] = rng.normal(0.0, 0.5, (n, 3))
    state[:, _abi.ST_QUAT:_abi.ST_QUAT + 4] = Rotation.random(n, random_state=rng).as_quat(scalar_first=True)
    state[:, _abi.ST_LINVEL:_abi.ST_LINVEL + 3] = rng.normal(0.0, 1.0, (n, 3))
    state[:, _abi.ST_ANGVEL:_abi.ST_ANGVEL + 3] = rng.normal(0.0, 2.0, (n, 3))
    state[:, _abi.ST_IMU_ACC:_abi.ST_IMU_ACC + 3] = rng.normal(0.0, 3.0, (n, 3))
    state[:, _abi.ST_Q:_abi.ST_Q + 6] = rng.normal(0.0, 0.5, (n, 6))
    state[:, _abi.ST_QD:_abi.ST_QD + 6] = rng.normal(0.0, 1.0, (n, 6))
    return state


def _obs(state, e):
    n = len(state)
    sim = _Sim()
    spine = np.zeros((n, _abi.SPINE_DIM), dtype=np.float32)
    o6 = np.zeros((n, 6), dtype=np.float32)
    changed = np.zeros(n, dtype=np.int32)
    _lib().hostsim_imu_misalign_obs(sim.h, n, _p(np.ascontiguousarray(state)),
                                    _p(np.ascontiguousarray(e, dtype=np.float32)), _p(spine), _p(o6), _p(changed, ip))
    return spine, o6, changed


def test_struct_matches_the_header():
    header = open(HEADER).read()
    body = re.search(r"typedef struct UpkieImuMisalignment \{(.*?)\} UpkieImuMisalignment;", header, re.S).group(1)
    names = re.findall(r"\b(\w+)\s*[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f[0] for f in _abi.UpkieImuMisalignment._fields_]
    assert C.sizeof(_abi.UpkieImuMisalignment) == 24


def test_draws_match_the_numpy_law():
    spec = _abi.UpkieImuMisalignment(-0.05, 0.02, -0.1, 0.1, 0.0, 0.3)
    g = np.arange(7, 71, dtype=np.uint64)
    for k in (1, 2, 1000, 2 ** 31 + 3):
        angles = angles_np(spec, SEED, g, k)
        for a, (lo, hi) in enumerate(((-0.05, 0.02), (-0.1, 0.1), (0.0, 0.3))):
            assert angles[:, a].min() >= np.float32(lo) and angles[:, a].max() <= np.float32(hi)
        ref = quat_np(angles)
        e = np.zeros(4, dtype=np.float32)
        got = np.zeros((len(g), 4))
        for j, x in enumerate(g):
            _lib().hostsim_imu_misalign_draw(C.byref(spec), SEED, int(x), k, _p(e))
            got[j] = e
        np.testing.assert_allclose(got, ref, atol=2e-7)
        np.testing.assert_allclose(np.linalg.norm(got, axis=1), 1.0, atol=1e-6)
    # distinct draws, and the draws of a degenerate range are that angle
    assert len(np.unique(angles_np(spec, SEED, g, 1)[:, 1])) == len(g)
    fixed = _abi.UpkieImuMisalignment(0.0, 0.0, 0.03, 0.03, 0.0, 0.0)
    np.testing.assert_array_equal(angles_np(fixed, SEED, g, 5)[:, 1], np.float32(0.03))


def test_reset_counts_and_stores_the_draw():
    n = 40
    spec = _abi.UpkieImuMisalignment(-0.02, 0.02, -0.04, 0.04, -0.1, 0.1)
    count = np.full(n, 4, dtype=np.uint32)
    quat = np.zeros((4, n), dtype=np.float32)
    _lib().hostsim_imu_misalign_reset(n, C.byref(spec), SEED, 100, _p(count, u32p), _p(quat))
    assert (count == 5).all()
    np.testing.assert_allclose(quat.T, quat_np(angles_np(spec, SEED, 100 + np.arange(n), 5)), atol=2e-7)
    # sharding: the draw is keyed on the global env index
    np.testing.assert_allclose(quat.T[20:], quat_np(angles_np(spec, SEED, 120 + np.arange(20), 5)), atol=2e-7)


@pytest.mark.parametrize("scale", [0.02, 0.3, 0.78])
def test_observations_are_those_of_the_tilted_imu(scale):
    rng = np.random.default_rng(int(scale * 100))
    n = 256
    state = random_states(n, rng)
    angles = rng.uniform(-scale, scale, (n, 3))
    e = quat_np(angles)
    spine, o6, changed = _obs(state, e)
    assert changed.all()
    ref = observe_np(state, e)
    check_spine(spine, ref)
    np.testing.assert_allclose(o6[:, 1], ref["pitch"], atol=2e-5)
    np.testing.assert_allclose(o6[:, 4], ref["base_angvel"][:, 1], atol=2e-4, rtol=1e-5)
    # not affected: the linear velocity (world frame), the servos, the odometry, the contact
    ident, o6_ident, unchanged = _obs(state, np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)))
    assert not unchanged.any()
    keep = [*range(_abi.SP_BASE_LINVEL, _abi.SP_BASE_LINVEL + 3), *range(_abi.SP_IMU_RAWACC + 3, _abi.SPINE_DIM)]
    np.testing.assert_array_equal(spine[:, keep], ident[:, keep])
    np.testing.assert_array_equal(o6[:, [0, 2, 3, 5]], o6_ident[:, [0, 2, 3, 5]])


def test_pure_pitch_offset_adds_to_the_pitch():
    rng = np.random.default_rng(3)
    n = 128
    state = random_states(n, rng)
    pitch = rng.uniform(-0.3, 0.3, n)
    state[:, _abi.ST_QUAT:_abi.ST_QUAT + 4] = Rotation.from_euler("ZYX", np.stack(
        [rng.uniform(-np.pi, np.pi, n), pitch, np.zeros(n)], axis=1)).as_quat(scalar_first=True)
    delta = rng.uniform(-0.1, 0.1, n)
    spine, o6, _ = _obs(state, quat_np(np.stack([np.zeros(n), delta, np.zeros(n)], axis=1)))
    np.testing.assert_allclose(o6[:, 1], pitch + delta, atol=3e-6)
    np.testing.assert_allclose(spine[:, _abi.SP_PITCH], pitch + delta, atol=3e-6)


def test_identity_leaves_the_state_bit_for_bit():
    n = 64
    state = random_states(n, np.random.default_rng(5))
    state[:8, _abi.ST_QUAT + 1] = -0.0  # a product with the identity would turn -0 into +0
    state[:8, _abi.ST_QUAT:_abi.ST_QUAT + 4] /= np.linalg.norm(state[:8, _abi.ST_QUAT:_abi.ST_QUAT + 4], axis=1,
                                                                keepdims=True)
    _, _, changed = _obs(state, np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)))
    assert not changed.any()
    # the smallest rotation is not the identity: w rounds to 1 below about 7e-4 rad
    _, _, changed = _obs(state, quat_np(np.tile([0.0, 1e-4, 0.0], (n, 1))))
    assert changed.all()


def _why(spec, limits=1, spine=0, body=0):
    buf = C.create_string_buffer(256)
    r = _lib().hostsim_imu_misalign_spec_error(C.byref(spec), limits, spine, body, buf, 256)
    return buf.value.decode() if r else None


def test_spec_rejections():
    ok = _abi.UpkieImuMisalignment(-0.1, 0.1, -0.2, 0.2, 0.0, 0.0)
    assert _why(ok) is None
    quarter = float(np.float32(np.pi / 4))
    assert _why(_abi.UpkieImuMisalignment(-quarter, quarter, 0, 0, 0, 0)) is None
    bad_bound = "set_imu_misalignment: every bound must be finite and within [-pi/4, pi/4] radians"
    for k in range(6):
        for v in (float("nan"), float("inf"), -float("inf"), 0.8, -0.8):
            b = [0.0] * 6
            b[k] = v
            if k % 2 == 0 and v > 0:
                b[k + 1] = v  # keep low <= high where the bound is finite
            assert _why(_abi.UpkieImuMisalignment(*b)) == bad_bound, (k, v)
    for k in range(0, 6, 2):
        b = [0.0] * 6
        b[k], b[k + 1] = 0.1, 0.05
        assert _why(_abi.UpkieImuMisalignment(*b)) == "set_imu_misalignment: low <= high required for roll, pitch and yaw"
    assert "joint_limits" in _why(ok, limits=0)
    assert "spine_mode" in _why(ok, spine=1)
    assert "body_contacts" in _why(ok, body=1)


def _family(limits=1, spine=0, body=0, obs_delay=0, mode=0, transport=0):
    buf = C.create_string_buffer(256)
    f = _lib().hostsim_step_family_imu_misalign(limits, spine, body, obs_delay, mode, transport, buf, 256)
    return f, buf.value.decode()


def test_family_choice():
    for mode in range(3):
        for transport in (0, 1):
            assert _family(mode=mode, transport=transport)[0] == FAM_SENSE
            assert _family(mode=mode, transport=transport, obs_delay=1)[0] == FAM_SENSE
    f, why = _family(transport=2)
    assert f == -1 and why == "IMU misalignment has no in-kernel rollout transport (use upkie_b200_step with compact rows)"
    assert _family(spine=1) == (-1, "IMU misalignment: spine_mode models its spine's own IMU")
    assert _family(limits=0) == (-1, "IMU misalignment needs joint_limits != 0")
    assert _family(body=1) == (-1, "IMU misalignment has no body-contact kernels")


def test_python_spec_validation():
    s = imu_misalignment_spec({"pitch": 0.05})
    assert (s.roll_low, s.roll_high, s.pitch_low, s.pitch_high, s.yaw_low, s.yaw_high) == \
        (0.0, 0.0, np.float32(0.05), np.float32(0.05), 0.0, 0.0)
    s = imu_misalignment_spec({"roll": (-0.01, 0.02), "yaw": (-0.3, 0.3)})
    assert (s.roll_low, s.roll_high, s.yaw_high) == (np.float32(-0.01), np.float32(0.02), np.float32(0.3))
    assert imu_misalignment_spec(None) is None
    assert imu_misalignment_spec({"pitch": (-np.pi / 4, np.pi / 4)}) is not None
    for bad in ({"pitch": (0.2, 0.1)}, {"roll": 0.9}, {"yaw": (-1.0, 0.0)}, {"pitch": float("nan")},
                {"pitch": (0.0, float("inf"))}, {"tilt": 0.1}, {"pitch": "x"}, {"pitch": (0.1, 0.2, 0.3)}, 0.1):
        with pytest.raises(UpkieException, match="imu_misalignment"):
            imu_misalignment_spec(bad)
    for kw in ({"spine_mode": True}, {"joint_limits": 0}, {"body_contacts": True}):
        with pytest.raises(UpkieException, match="imu_misalignment"):
            imu_misalignment_spec({"pitch": 0.01}, **kw)
