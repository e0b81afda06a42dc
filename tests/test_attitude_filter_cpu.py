# SPDX-License-Identifier: Apache-2.0
"""IMU attitude estimation (upkie_b200_set_attitude_filter): the C struct against its mirror; the draw law compiled
for the CPU (tests/hostsim/attitude_filter.cpp) against a NumPy statement of include/upkie_b200.h; the filter step
against an fp64 restatement, over random inputs and long synthetic sequences; the analytic behaviour of the law
(convergence at exp(-kp t), the tilt error of a gyro bias and of a horizontal acceleration, the bias estimate, the
unobservable yaw) on both; the initial estimate and the observation read from an estimate; the spec's validation on
both sides and the family choice. No GPU needed."""
import ctypes as C
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from upkie_b200 import UpkieException, _abi
from upkie_b200.envs import attitude_filter_spec
from upkie_b200.model import default_model
from test_reset_randomization_cpu import philox_np

HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(HERE, "..", "include", "upkie_b200.h")
FAM_SENSE = 10
G = 9.81
H = 0.001  # the substep of the default 200 Hz / 5 substeps
RBI = np.diag([-1.0, 1.0, -1.0])  # rotation_base_to_imu of the default model

_LIB = None
fp = C.POINTER(C.c_float)


def _lib():
    global _LIB
    if _LIB is None:
        src = os.path.join(HERE, "hostsim", "attitude_filter.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_att_"), "libhostsim_attitude_filter.so")
        flags = os.environ.get("UPKIE_HOSTSIM_CXXFLAGS", "-O2").split()
        subprocess.check_call(["g++", *flags, "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp = C.c_void_p
        spec_p = C.POINTER(_abi.UpkieAttitudeFilter)
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_att_draw.argtypes = [spec_p, C.c_uint64, C.c_uint64, C.c_uint32, fp]
        L.hostsim_att_run.argtypes = [C.c_int, fp, fp, C.c_float, C.c_float, C.c_float, fp, fp, C.c_int, fp, fp]
        L.hostsim_att_inputs.argtypes = [vp, C.c_int, fp, fp, fp, fp, fp, fp, fp]
        L.hostsim_att_initial.argtypes = [vp, C.c_int, fp, fp, fp, fp]
        L.hostsim_att_observation.argtypes = [vp, C.c_int, fp, fp, fp]
        L.hostsim_att_spec_error.argtypes = [spec_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_char_p, C.c_int]
        L.hostsim_step_family_att.argtypes = [C.c_int] * 5 + [C.c_char_p, C.c_int]
        _LIB = L
    return _LIB


def _p(a):
    return a.ctypes.data_as(fp)


@pytest.fixture(scope="module")
def hs():
    L = _lib()
    m, c = default_model().to_struct(), _abi.default_sim_config()
    h = L.hostsim_create(C.byref(m), C.byref(c))
    assert h
    yield h
    L.hostsim_destroy(h)


def u01(w):
    return (np.asarray(w, dtype=np.uint32) >> np.uint32(8)).astype(np.float32) * np.float32(1.0 / 16777216.0)


def draw_np(spec, seed, g, k):
    """[len(g), 4] kp, ki, roll, pitch of draw k of the envs of global index g (include/upkie_b200.h): fp32, the
    product rounded on its own, clamped to high"""
    g = np.atleast_1d(np.asarray(g, dtype=np.uint64))
    hi = np.uint64(1 << 51) | (np.broadcast_to(np.asarray(k, dtype=np.uint64), g.shape) << np.uint64(4))
    w = philox_np(g, hi, np.full(g.shape, seed, dtype=np.uint64))
    out = np.zeros(g.shape + (4,), dtype=np.float32)
    for a, key in enumerate(("kp", "ki", "roll", "pitch")):
        lo, high = np.float32(getattr(spec, key + "_low")), np.float32(getattr(spec, key + "_high"))
        out[:, a] = np.minimum(lo + (high - lo) * u01(w[a]), high)
    return out


def qmul(p, q):
    w1, x1, y1, z1 = p
    w2, x2, y2, z2 = q
    return np.array([w1 * w2 - x1 * x2 - y1 * y2 - z1 * z2, w1 * x2 + x1 * w2 + y1 * z2 - z1 * y2,
                     w1 * y2 - x1 * z2 + y1 * w2 + z1 * x2, w1 * z2 + x1 * y2 - y1 * x2 + z1 * w2])


def step_np(q, b, kp, ki, h, wm, am):
    """One step of the law of include/upkie_b200.h in fp64 (exact cos and sin)"""
    w, x, y, z = q
    v = np.array([2 * (x * z - y * w), 2 * (y * z + x * w), 1 - 2 * (x * x + y * y)])
    n = np.linalg.norm(am)
    e = np.cross(am / n, v) if n > 1e-3 else np.zeros(3)
    b = b - ki * e * h
    om = wm - b + kp * e
    nw = np.linalg.norm(om)
    if nw > 0:
        t = 0.5 * nw * h
        q = qmul(q, np.concatenate([[np.cos(t)], np.sin(t) / nw * om]))
        q = q / np.linalg.norm(q)
    return q, b


def run_np(q, b, kp, ki, h, wm, am, steps):
    wm, am = np.broadcast_to(wm, (steps, 3)), np.broadcast_to(am, (steps, 3))
    qs, bs = np.zeros((steps, 4)), np.zeros((steps, 3))
    q, b = np.asarray(q, float), np.asarray(b, float)
    for s in range(steps):
        q, b = step_np(q, b, kp, ki, h, wm[s], am[s])
        qs[s], bs[s] = q, b
    return qs, bs


def run_hs(q, b, kp, ki, h, wm, am, steps):
    """the same with the kernels' arithmetic (fp32); an input of one row repeats for every step"""
    q = np.array(q, dtype=np.float32)
    b = np.array(b, dtype=np.float32)
    wm = np.ascontiguousarray(np.atleast_2d(wm), dtype=np.float32)
    am = np.ascontiguousarray(np.atleast_2d(am), dtype=np.float32)
    stride = 0 if len(wm) == 1 else 3
    qs, bs = np.zeros((steps, 4), np.float32), np.zeros((steps, 3), np.float32)
    _lib().hostsim_att_run(steps, _p(q), _p(b), kp, ki, h, _p(wm), _p(am), stride, _p(qs), _p(bs))
    return qs.astype(np.float64), bs.astype(np.float64)


RUNS = {"numpy_fp64": run_np, "hostsim": run_hs}


def up(q):
    """R(q)^T e_z, the world's up in the IMU frame of an IMU-to-world rotation q"""
    return Rotation.from_quat(q, scalar_first=True).inv().apply([0.0, 0.0, 1.0])


def tilt_error(q_est, q_true):
    return np.arccos(np.clip(np.dot(up(q_est), up(q_true)), -1.0, 1.0))


def spec_of(kp=(1.0, 1.0), ki=(0.0, 0.0), roll=(0.0, 0.0), pitch=(0.0, 0.0)):
    return _abi.UpkieAttitudeFilter(*kp, *ki, *roll, *pitch)


def test_struct_matches_the_header():
    with open(HEADER) as f:
        text = f.read()
    body = re.search(r"typedef struct UpkieAttitudeFilter \{(.*?)\} UpkieAttitudeFilter;", text, re.S).group(1)
    names = re.findall(r"(\w+)[,;]", re.sub(r"/\*.*?\*/", "", body, flags=re.S))
    assert names == [f for f, _ in _abi.UpkieAttitudeFilter._fields_]
    assert C.sizeof(_abi.UpkieAttitudeFilter) == 32


def test_draws_match_the_numpy_law():
    L = _lib()
    spec = spec_of((1.0, 10.0), (0.0, 0.5), (-0.05, 0.05), (-0.2, 0.1))
    rng = np.random.default_rng(3)
    out = np.zeros(4, np.float32)
    for _ in range(300):
        seed, g, k = int(rng.integers(0, 2**63)), int(rng.integers(0, 2**40)), int(rng.integers(0, 2**32))
        L.hostsim_att_draw(C.byref(spec), seed, g, k, _p(out))
        assert np.array_equal(out, draw_np(spec, seed, g, k)[0])
        assert spec.kp_low <= out[0] <= spec.kp_high and spec.ki_low <= out[1] <= spec.ki_high


@pytest.mark.parametrize("field", ["kp", "ki", "roll", "pitch"])
def test_one_range_changes_no_other_word(field):
    L = _lib()
    base = spec_of((1.0, 10.0), (0.0, 0.5), (-0.05, 0.05), (-0.05, 0.05))
    other = spec_of((1.0, 10.0), (0.0, 0.5), (-0.05, 0.05), (-0.05, 0.05))
    setattr(other, field + "_high", getattr(other, field + "_high") * 0.5)
    a, b = np.zeros(4, np.float32), np.zeros(4, np.float32)
    col = ("kp", "ki", "roll", "pitch").index(field)
    for g in range(50):
        L.hostsim_att_draw(C.byref(base), 9, g, 3, _p(a))
        L.hostsim_att_draw(C.byref(other), 9, g, 3, _p(b))
        keep = [c for c in range(4) if c != col]
        assert np.array_equal(a[keep], b[keep])


def test_step_matches_fp64_over_random_inputs():
    rng = np.random.default_rng(5)
    for _ in range(500):
        q = Rotation.random(random_state=rng).as_quat(scalar_first=True)
        b = rng.normal(0, 0.05, 3)
        wm = rng.normal(0, 3.0, 3)
        am = rng.normal(0, 3.0, 3) + up(q) * G
        kp, ki = rng.uniform(0, 400), rng.uniform(0, 10)
        qn, bn = run_np(q, b, kp, ki, H, wm, am, 1)
        qh, bh = run_hs(q, b, kp, ki, H, wm, am, 1)
        assert np.abs(qh - qn).max() < 2e-6 and np.abs(bh - bn).max() < 2e-6


def test_large_rotation_step_matches_fp64():
    # |w| h / 2 >= 0.25: cos and sin instead of the series
    q = np.array([1.0, 0.0, 0.0, 0.0])
    for wm in ([600.0, 0.0, 0.0], [300.0, -500.0, 200.0]):
        qn, _ = run_np(q, np.zeros(3), 0.0, 0.0, H, np.array(wm), np.array([0, 0, G]), 1)
        qh, _ = run_hs(q, np.zeros(3), 0.0, 0.0, H, np.array(wm), np.array([0, 0, G]), 1)
        assert np.abs(qh - qn).max() < 2e-6


def test_long_sequences_match_fp64():
    rng = np.random.default_rng(11)
    steps = 10_000
    t = np.arange(steps) * H
    for trial in range(2):
        # a swaying, accelerating IMU with a biased gyro: the rate and specific force of a synthetic trajectory
        f = rng.uniform(0.2, 2.0, 3)
        wm = np.stack([0.8 * np.sin(2 * np.pi * f[k] * t + k) for k in range(3)], 1) + rng.normal(0, 0.01, 3)
        am = np.stack([1.5 * np.sin(2 * np.pi * f[1] * t), 0.7 * np.cos(2 * np.pi * f[2] * t), np.full(steps, G)], 1)
        q0 = Rotation.from_euler("xyz", rng.uniform(-0.3, 0.3, 3)).as_quat(scalar_first=True)
        kp, ki = [(5.0, 0.3), (40.0, 2.0)][trial]
        qn, bn = run_np(q0, np.zeros(3), kp, ki, H, wm, am, steps)
        qh, bh = run_hs(q0, np.zeros(3), kp, ki, H, wm, am, steps)
        sign = np.sign(np.sum(qn * qh, axis=1, keepdims=True))
        assert np.abs(qh * sign - qn).max() < 5e-5
        assert np.abs(bh - bn).max() < 5e-5


@pytest.mark.parametrize("run", list(RUNS))
def test_still_imu_error_decays_at_kp(run):
    kp, theta, e0 = 4.0, 0.3, 0.02
    q_true = Rotation.from_euler("y", theta).as_quat(scalar_first=True)
    q0 = (Rotation.from_euler("y", theta) * Rotation.from_euler("x", e0)).as_quat(scalar_first=True)
    am = up(q_true) * G
    steps = 500
    qs, _ = RUNS[run](q0, np.zeros(3), kp, 0.0, H, np.zeros(3), am, steps)
    err0 = tilt_error(q0, q_true)  # e0 about the tilted x axis: e0 cos(theta) of tilt
    for s in (99, 249, 499):
        expected = err0 * np.exp(-kp * (s + 1) * H)
        assert tilt_error(qs[s], q_true) == pytest.approx(expected, rel=0.03, abs=2e-6)


@pytest.mark.parametrize("run", list(RUNS))
def test_gyro_bias_tilt_error_and_bias_estimate(run):
    bias = np.array([0.02, -0.01, 0.0])
    q_true = np.array([1.0, 0.0, 0.0, 0.0])
    am = np.array([0.0, 0.0, G])
    kp = 2.0
    # ki = 0: the steady tilt error is |b| / kp
    qs, _ = RUNS[run](q_true, np.zeros(3), kp, 0.0, H, bias, am, 5000)
    assert tilt_error(qs[-1], q_true) == pytest.approx(np.linalg.norm(bias) / kp, rel=0.02)
    # ki > 0: the bias estimate converges to b and the tilt error to 0
    qs, bs = RUNS[run](q_true, np.zeros(3), kp, 1.0, H, bias, am, 20_000)
    assert np.abs(bs[-1] - bias).max() < 2e-4
    assert tilt_error(qs[-1], q_true) < 2e-4


@pytest.mark.parametrize("run", list(RUNS))
def test_horizontal_specific_force_tilts_by_atan(run):
    a = 2.0
    q_true = np.array([1.0, 0.0, 0.0, 0.0])
    am = np.array([a, 0.0, G])
    qs, _ = RUNS[run](q_true, np.zeros(3), 10.0, 0.0, H, np.zeros(3), am, 3000)
    assert tilt_error(qs[-1], q_true) == pytest.approx(np.arctan(a / G), rel=1e-3)


@pytest.mark.parametrize("run", list(RUNS))
def test_yaw_drifts_at_the_z_bias(run):
    bz = 0.05
    q_true = np.array([1.0, 0.0, 0.0, 0.0])
    steps = 2000
    qs, _ = RUNS[run](q_true, np.zeros(3), 5.0, 1.0, H, np.array([0.0, 0.0, bz]), np.array([0.0, 0.0, G]), steps)
    yaw = Rotation.from_quat(qs[-1], scalar_first=True).as_euler("ZYX")[0]
    assert yaw == pytest.approx(bz * steps * H, rel=1e-3)
    assert tilt_error(qs[-1], q_true) < 1e-6


def test_inputs_are_the_imu_frame_rate_and_specific_force(hs):
    rng = np.random.default_rng(2)
    n = 16
    state = np.zeros((n, _abi.STATE_DIM), np.float32)
    qb = Rotation.random(n, random_state=rng).as_quat(scalar_first=True)
    state[:, 3:7] = qb
    state[:, 7:10] = rng.normal(0, 1, (n, 3))   # linear velocity
    state[:, 10:13] = rng.normal(0, 2, (n, 3))  # angular velocity (world frame)
    vp = rng.normal(0, 1, (n, 3)).astype(np.float32)
    gb = np.array([0.01, -0.02, 0.03], np.float32)
    ab = np.array([0.1, 0.0, -0.1], np.float32)
    v, wm, am = (np.zeros((n, 3), np.float32) for _ in range(3))
    _lib().hostsim_att_inputs(hs, n, _p(state), _p(vp), _p(gb), _p(ab), _p(v), _p(wm), _p(am))
    imu_pos = np.asarray(default_model().imu_position, dtype=np.float64)
    for i in range(n):
        Rb = Rotation.from_quat(qb[i], scalar_first=True).as_matrix()
        Ri = Rb @ RBI.T
        vi = state[i, 7:10] + np.cross(state[i, 10:13], Rb @ imu_pos)
        assert np.allclose(v[i], vi, atol=1e-5)
        assert np.allclose(wm[i], Ri.T @ state[i, 10:13] + gb, atol=1e-5)
        f = (v[i].astype(np.float64) - vp[i]) / H + [0, 0, G]
        assert np.allclose(am[i], Ri.T @ f + ab, rtol=1e-5, atol=2e-3)


def test_initial_estimate_and_its_observation(hs):
    rng = np.random.default_rng(4)
    n = 32
    qb = Rotation.from_euler("xyz", rng.uniform(-0.5, 0.5, (n, 3))).as_quat(scalar_first=True).astype(np.float32)
    roll = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    pitch = rng.uniform(-0.1, 0.1, n).astype(np.float32)
    q = np.zeros((n, 4), np.float32)
    _lib().hostsim_att_initial(hs, n, _p(qb), _p(roll), _p(pitch), _p(q))
    o = np.zeros((n, _abi.SPINE_DIM), np.float32)
    pit = np.zeros(n, np.float32)
    _lib().hostsim_att_observation(hs, n, _p(q), _p(o), _p(pit))
    for i in range(n):
        Rest = (Rotation.from_quat(qb[i], scalar_first=True) * Rotation.from_euler("ZYX", [0, pitch[i], roll[i]]))
        # the estimate is an IMU-to-world rotation: taken back to the base through rotation_base_to_imu
        Ri = Rotation.from_quat(q[i], scalar_first=True).as_matrix()
        assert np.allclose(Ri @ RBI, Rest.as_matrix(), atol=2e-6)
        R = Rest.as_matrix()
        assert np.allclose(o[i, _abi.SP_ROT:_abi.SP_ROT + 9], R.reshape(-1), atol=2e-6)
        assert o[i, _abi.SP_PITCH] == pytest.approx(np.arcsin(-R[2, 0]), abs=2e-6)
        assert pit[i] == o[i, _abi.SP_PITCH]
        ars = np.diag([1.0, -1.0, -1.0]) @ R @ RBI.T
        qa = Rotation.from_matrix(ars).as_quat(scalar_first=True)
        got = o[i, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4]
        assert min(np.abs(got - qa).max(), np.abs(got + qa).max()) < 2e-6


def _why(spec, limits=1, spine=0, body=0, h=H):
    buf = C.create_string_buffer(256)
    bad = _lib().hostsim_att_spec_error(C.byref(spec), limits, spine, body, h, buf, 256)
    return buf.value.decode() if bad else None


def test_spec_rejections():
    assert _why(spec_of((1.0, 10.0), (0.0, 0.5), (-0.05, 0.05), (-0.05, 0.05))) is None
    assert _why(spec_of((0.0, 499.0))) is None  # kp_high * h just below 0.5
    bad = {
        "finite": spec_of((1.0, float("nan"))),
        "inf": spec_of((1.0, 1.0), (0.0, float("inf"))),
        "low <= high": spec_of((2.0, 1.0)),
        "kp_low >= 0": spec_of((-1.0, 1.0)),
        "<= 0.5": spec_of((1.0, 501.0)),
        "ki_low": spec_of((1.0, 1.0), (-0.1, 0.0)),
        "ki_high": spec_of((1.0, 1.0), (0.0, 10.5)),
        "roll": spec_of(roll=(-0.8, 0.0)),
        "pitch": spec_of(pitch=(0.0, 0.8)),
    }
    for what, spec in bad.items():
        assert _why(spec) is not None, what
    ok = spec_of()
    assert "joint_limits" in _why(ok, limits=0)
    assert "spine_mode" in _why(ok, spine=1)
    assert "body_contacts" in _why(ok, body=1)
    assert _why(spec_of((1.0, 200.0)), h=0.005) is not None  # 200 * 5 ms > 0.5: a coarser substep refuses it


def test_family_choice():
    buf = C.create_string_buffer(256)
    L = _lib()
    for mode in (0, 1, 2):
        assert L.hostsim_step_family_att(1, 0, 0, mode, 0, buf, 256) == FAM_SENSE
        assert L.hostsim_step_family_att(2, 0, 0, mode, 1, buf, 256) == FAM_SENSE
    assert L.hostsim_step_family_att(1, 0, 0, 0, 2, buf, 256) == -1
    assert b"attitude filter" in buf.value
    for args in ((0, 0, 0), (1, 1, 0), (1, 0, 1)):
        assert L.hostsim_step_family_att(*args, 0, 0, buf, 256) == -1


def test_python_spec_validation():
    spec = attitude_filter_spec({"kp": (1.0, 10.0), "ki": (0.0, 0.5), "roll": (-0.05, 0.05), "pitch": 0.02})
    assert (spec.kp_low, spec.kp_high, spec.pitch_low, spec.pitch_high) == (1.0, 10.0, np.float32(0.02),
                                                                            np.float32(0.02))
    assert attitude_filter_spec(None) is None
    bad = [
        {"ki": 0.1},  # kp is required
        {"kp": 1.0, "yaw": 0.1},
        {"kp": (2.0, 1.0)},
        {"kp": -1.0},
        {"kp": float("nan")},
        {"kp": 1.0, "ki": 11.0},
        {"kp": 1.0, "ki": (-0.1, 0.0)},
        {"kp": 1.0, "roll": 0.9},
        {"kp": 1.0, "pitch": (-1.0, 0.0)},
        {"kp": "fast"},
        [1.0, 2.0],
    ]
    for b in bad:
        with pytest.raises(UpkieException):
            attitude_filter_spec(b)
    with pytest.raises(UpkieException):
        attitude_filter_spec({"kp": 600.0}, dt=1 / 200, nb_substeps=5)
    attitude_filter_spec({"kp": 499.0}, dt=1 / 200, nb_substeps=5)
    for kw in ({"spine_mode": True}, {"joint_limits": False}, {"body_contacts": True}, {"obs_delay_ticks": 2}):
        with pytest.raises(UpkieException):
            attitude_filter_spec({"kp": 1.0}, **kw)
