# SPDX-License-Identifier: Apache-2.0
"""Per-env parameter table (upkie_b200_set_env_params): layout, the B200VectorEnv argument forms, validation and
forwarding, and the kernels' arithmetic with a table on the CPU build (tests/hostsim). No GPU needed."""
import ctypes as C
import os
import re
import sys
import types

import numpy as np
import pytest

from upkie_b200 import JointProperties, UpkieException, _abi

N = 6
JOINTS = _abi.JOINT_NAMES


def test_offsets_and_abi_match_the_header():
    header = open(os.path.join(os.path.dirname(__file__), "..", "include", "upkie_b200.h")).read()
    defs = dict(re.findall(r"#define (UPKIE_\w+) (\d+)", header))
    assert int(defs["UPKIE_B200_ABI_VERSION"]) == _abi.ABI_VERSION == 8
    for name in ("KP", "KD", "FRICTION", "CTRL_NOISE", "MEAS_NOISE", "IMU_ACC_BIAS", "IMU_ACC_NOISE", "IMU_GYRO_BIAS",
                 "IMU_GYRO_NOISE", "DIM"):
        assert int(defs[f"UPKIE_EP_{name}"]) == getattr(_abi, f"EP_{name}"), name


class _FakeSim:
    """Stands in for UpkieSim: records the config and the table B200VectorEnv hands it."""

    def __init__(self, n, model=None, config=None, device=0):
        self.n, self.config, self.device, self.env_params = n, config, "cpu", None

    def set_autoreset(self, *args):
        pass

    def set_env_params(self, rows):
        self.env_params = None if rows is None else rows.numpy().copy()

    def get_env_params(self):
        import torch

        rows = self.env_params if self.env_params is not None else np.tile(_abi.config_env_params(self.config), (self.n, 1))
        return torch.from_numpy(rows)


@pytest.fixture
def fake_sim(monkeypatch):
    from upkie_b200 import envs

    monkeypatch.setattr(envs, "UpkieSim", _FakeSim)
    return envs


def test_scalar_arguments_build_no_table_and_todays_config(fake_sim):
    props = {"left_hip": JointProperties(0.1, 0.02, 0.03), "right_wheel": JointProperties(friction=0.2)}
    env = fake_sim.B200VectorEnv(N, "servos", torque_control_kp=25.0, torque_control_kd=0.5, joint_properties=props)
    assert env.sim.env_params is None
    today = fake_sim.make_config(200.0, None, 25.0, 0.5, props, init_state=env.init_state)
    assert bytes(env.config) == bytes(today)


def test_array_gains_and_array_joint_properties(fake_sim):
    kp = np.linspace(15.0, 25.0, N)
    fr = np.linspace(0.0, 0.05, N)
    props = {"left_knee": JointProperties(friction=fr, torque_control_noise=0.01), "right_hip": JointProperties(0.3)}
    env = fake_sim.B200VectorEnv(N, "servos", torque_control_kp=kp, torque_control_kd=0.7, joint_properties=props)
    t = env.sim.env_params
    assert t.shape == (N, _abi.EP_DIM) and t.dtype == np.float32 and t.flags["C_CONTIGUOUS"]
    row = _abi.config_env_params(env.config)
    expect = np.tile(row, (N, 1))
    expect[:, _abi.EP_KP] = kp.astype(np.float32)
    expect[:, _abi.EP_KD] = np.float32(0.7)
    expect[:, _abi.EP_FRICTION + 1] = fr.astype(np.float32)
    expect[:, _abi.EP_CTRL_NOISE + 1] = np.float32(0.01)
    expect[:, _abi.EP_FRICTION + 3] = np.float32(0.3)
    np.testing.assert_array_equal(t, expect)
    # the config keeps the scalar defaults of what went to the table
    assert env.config.torque_control_kp == 20.0 and list(env.config.joint_friction) == [0.0] * 6


def test_list_of_per_env_dicts(fake_sim):
    dicts = [{"left_wheel": JointProperties(friction=0.01 * i, torque_measurement_noise=0.001 * i)} for i in range(N)]
    env = fake_sim.B200VectorEnv(N, "servos", joint_properties=dicts)
    t = env.sim.env_params
    np.testing.assert_array_equal(t[:, _abi.EP_FRICTION + 2], np.float32(0.01 * np.arange(N)))
    np.testing.assert_array_equal(t[:, _abi.EP_MEAS_NOISE + 2], np.float32(0.001 * np.arange(N)))
    np.testing.assert_array_equal(t[:, _abi.EP_KP], np.float32(20.0))
    np.testing.assert_array_equal(t[:, _abi.EP_FRICTION], 0.0)


def test_set_joint_properties_keeps_what_is_not_given(fake_sim):
    env = fake_sim.B200VectorEnv(N, "servos", torque_control_kp=np.full(N, 18.0))
    env.set_joint_properties({"left_hip": JointProperties(friction=np.arange(N) * 0.01)}, torque_control_kd=1.5)
    t = env.sim.env_params
    np.testing.assert_array_equal(t[:, _abi.EP_KP], np.float32(18.0))
    np.testing.assert_array_equal(t[:, _abi.EP_KD], np.float32(1.5))
    np.testing.assert_array_equal(t[:, _abi.EP_FRICTION], np.float32(np.arange(N) * 0.01))


@pytest.mark.parametrize("kwargs", [
    {"torque_control_kp": np.ones(N - 1)},
    {"torque_control_kd": np.array([1.0, np.nan, 1.0, 1.0, 1.0, 1.0])},
    {"torque_control_kp": np.array([20.0, -1.0, 20.0, 20.0, 20.0, 20.0])},
    {"joint_properties": {"left_hip": JointProperties(friction=-np.ones(N))}},
    {"joint_properties": {"left_hip": JointProperties(torque_control_noise=np.full(N, -0.1))}},
    {"joint_properties": {"left_hip": JointProperties(torque_measurement_noise=np.full(N, np.inf))}},
    {"joint_properties": [{"left_hip": JointProperties()}] * (N + 1)},
])
def test_invalid_per_env_arguments_are_rejected_before_the_device(kwargs):
    from upkie_b200.envs import B200VectorEnv, env_params_table

    with pytest.raises(UpkieException):
        env_params_table(N, np.zeros(_abi.EP_DIM, np.float32), **kwargs)
    with pytest.raises(UpkieException):
        B200VectorEnv(N, "servos", **kwargs)  # no device on the build machine: rejected before it is needed


class _Recorder:
    calls = []

    def __init__(self, num_envs, env_type, **kwargs):
        _Recorder.calls.append((num_envs, env_type, kwargs))


def test_make_vec_and_register_forward_the_arguments(monkeypatch):
    import upkie_b200
    from upkie_b200 import envs

    kp = np.full(8, 22.0)
    props = [{"left_hip": JointProperties(0.1)}] * 8
    _Recorder.calls.clear()
    monkeypatch.setattr(envs, "B200VectorEnv", _Recorder)
    upkie_b200.make_vec("Upkie-B200-Servos", 8, torque_control_kp=kp, joint_properties=props)
    assert _Recorder.calls[-1][2]["torque_control_kp"] is kp and _Recorder.calls[-1][2]["joint_properties"] is props

    registered = {}
    gym = types.ModuleType("gymnasium")
    gym.registry = {}
    gym.register = lambda id, vector_entry_point: registered.__setitem__(id, vector_entry_point)
    monkeypatch.setitem(sys.modules, "gymnasium", gym)
    upkie_b200.register()
    registered["Upkie-B200-Servos"](num_envs=16, torque_control_kd=kp)
    assert _Recorder.calls[-1][2] == {"torque_control_kd": kp}


# ---- the kernels' arithmetic on the CPU (tests/hostsim/env_params.cpp) ---------------------------------------------------------


_EP_LIB = None


def _ep_lib():
    """tests/hostsim/env_params.cpp (the CPU build of the kernel arithmetic with the table's entry points), compiled
    into a temporary directory"""
    global _EP_LIB
    if _EP_LIB is None:
        import subprocess
        import tempfile

        src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim", "env_params.cpp")
        out = os.path.join(tempfile.mkdtemp(prefix="upkie_ep_"), "libhostsim_env_params.so")
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", out, src])
        L = C.CDLL(out)
        vp, fp, u32, u64, i32 = C.c_void_p, C.POINTER(C.c_float), C.c_uint32, C.c_uint64, C.c_int
        L.hostsim_create.restype = vp
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [vp]
        L.hostsim_reset.argtypes = [vp, i32, fp, fp, fp, fp]
        L.hostsim_sample_init.argtypes = [vp, i32, u64, u64, u64, fp]
        L.hostsim_reset_spine.argtypes = [vp, i32, fp, fp, fp, fp]
        L.hostsim_ep_set_env_params.argtypes = [vp, i32, fp, fp]
        L.hostsim_ep_set_env_params.restype = u32
        L.hostsim_ep_step_servos_noise.argtypes = [vp, i32, fp, fp, u32, u64, fp]
        L.hostsim_ep_spine_obs_with_uncertainty.argtypes = [vp, i32, fp, u32, u64, fp]
        L.hostsim_ep_step_servos_spine.argtypes = [vp, i32, fp, fp, fp, fp]
        _EP_LIB = L
    return _EP_LIB


def _f(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


class _EpSim:
    """n robots of the CPU build, one after the other, env i reading column i of the table when one is set"""

    def __init__(self, cfg, n):
        from upkie_b200.model import default_model

        self.L, self.n = _ep_lib(), n
        self._m = default_model().to_struct()
        self._c = cfg
        self._h = self.L.hostsim_create(C.byref(self._m), C.byref(cfg))
        assert self._h
        self.state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
        self.lag = np.zeros((n, _abi.LAG_DIM), dtype=np.float32)
        self._soa = np.zeros((_abi.EP_DIM, n), dtype=np.float32)  # the installed table (kept alive here)

    def __del__(self):
        try:
            self.L.hostsim_destroy(self._h)
        except Exception:
            pass

    def set_env_params(self, rows):
        rows = np.ascontiguousarray(rows, dtype=np.float32)
        return self.L.hostsim_ep_set_env_params(self._h, self.n, _f(rows), _f(self._soa))

    def sample_init(self, seed, env_offset):
        out = np.empty((self.n, _abi.INIT_DIM), dtype=np.float32)
        self.L.hostsim_sample_init(self._h, self.n, seed, env_offset, 1, _f(out))
        return out

    def reset(self, init):
        self.L.hostsim_reset(self._h, self.n, _f(self.state), _f(init), None, None)

    def step_servos_noise(self, action, tick, env_offset):
        a = np.ascontiguousarray(action, dtype=np.float32)
        obs = np.empty((self.n, 6, 5), dtype=np.float32)
        self.L.hostsim_ep_step_servos_noise(self._h, self.n, _f(self.state), _f(a), tick, env_offset, _f(obs))
        return obs

    def spine_obs_with_uncertainty(self, tick, env_offset):
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        self.L.hostsim_ep_spine_obs_with_uncertainty(self._h, self.n, _f(self.state), tick, env_offset, _f(out))
        return out

    def reset_spine(self, init):
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        self.L.hostsim_reset_spine(self._h, self.n, _f(self.state), _f(self.lag), _f(init), _f(out))
        return out

    def step_servos_spine(self, action):
        a = np.ascontiguousarray(action, dtype=np.float32)
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        self.L.hostsim_ep_step_servos_spine(self._h, self.n, _f(self.state), _f(self.lag), _f(a), _f(out))
        return out


def _config(kp=20.0, kd=1.0, friction=0.0, ctrl=0.0, meas=0.0, imu=0.0):
    cfg = _abi.default_sim_config()
    cfg.noise_seed = 77
    cfg.torque_control_kp, cfg.torque_control_kd = kp, kd
    for j in range(6):
        cfg.joint_friction[j] = friction * (1 + 0.1 * j)
        cfg.torque_control_noise[j] = ctrl
        cfg.torque_measurement_noise[j] = meas
    for k in range(3):
        cfg.imu_accelerometer_bias[k] = imu * (k - 1)
        cfg.imu_gyroscope_bias[k] = 0.5 * imu * k
    cfg.imu_accelerometer_noise, cfg.imu_gyroscope_noise = imu, 0.3 * imu
    return cfg


GROUPS = [_config(), _config(15.0, 0.6, 0.02, 0.03, 0.01, 0.05), _config(25.0, 1.4, 0.05, 0.0, 0.02, 0.0),
          _config(18.0, 1.1, 0.0, 0.05, 0.0, 0.1)]
PER = 2  # envs per group


def _actions(n, k, env_offset=0):
    """actions of tick k for the envs [env_offset, env_offset + n) of the whole batch"""
    total = PER * len(GROUPS)
    rng = np.random.default_rng(100 + k)
    a = np.zeros((total, 6, 6), dtype=np.float32)
    a[:, :, 0] = rng.uniform(-0.3, 0.3, (total, 6))  # position targets
    a[:, :, 1] = rng.uniform(-2.0, 2.0, (total, 6))  # velocity targets: kd and friction act
    a[:, :, 3] = a[:, :, 4] = 1.0
    a[:, :, 5] = 16.0
    return a[env_offset : env_offset + n]


def _run(cfg, n, env_offset, rows=None, ticks=6):
    """servo ticks with the noise models (k_step's sequence), then the spine observation with its uncertainty"""
    hs = _EpSim(cfg, n)
    if rows is not None:
        assert not (hs.set_env_params(rows) & 1)
    hs.reset(hs.sample_init(5, env_offset))  # keyed on the global env index, as the device sampler
    obs = [hs.step_servos_noise(_actions(n, t, env_offset), t + 1, env_offset) for t in range(ticks)]
    obs.append(hs.spine_obs_with_uncertainty(ticks, env_offset))
    obs.append(hs.state.copy())
    return obs


def test_hostsim_config_equal_table_is_bit_identical():
    cfg = GROUPS[1]
    n = 4
    plain = _run(cfg, n, 0)
    table = _run(cfg, n, 0, np.tile(_abi.config_env_params(cfg), (n, 1)))
    for a, b in zip(plain, table):
        np.testing.assert_array_equal(a, b)


def test_hostsim_heterogeneous_table_matches_grouped_configs():
    rows = np.concatenate([np.tile(_abi.config_env_params(c), (PER, 1)) for c in GROUPS])
    # a base config whose own values differ from every group: the table must override all of them
    mixed = _run(_config(30.0, 2.0, 0.1, 0.1, 0.1, 0.2), PER * len(GROUPS), 0, rows)
    for g, cfg in enumerate(GROUPS):
        alone = _run(cfg, PER, PER * g)
        for a, b in zip(mixed, alone):
            np.testing.assert_array_equal(a[PER * g : PER * (g + 1)], b)
    # the groups really differ
    assert not np.array_equal(mixed[-1][:PER], mixed[-1][PER : 2 * PER])


def test_hostsim_spine_mode_uses_the_gain_columns():
    def spine_run(cfg, n, env_offset, rows=None):
        hs = _EpSim(cfg, n)
        if rows is not None:
            assert not (hs.set_env_params(rows) & 1)
        out = [hs.reset_spine(hs.sample_init(9, env_offset))]
        out += [hs.step_servos_spine(_actions(n, t, env_offset)) for t in range(4)]
        return out

    rows = np.concatenate([np.tile(_abi.config_env_params(c), (PER, 1)) for c in GROUPS])
    mixed = spine_run(_config(), PER * len(GROUPS), 0, rows)
    for g, cfg in enumerate(GROUPS):
        for a, b in zip(mixed, spine_run(cfg, PER, PER * g)):
            np.testing.assert_array_equal(a[PER * g : PER * (g + 1)], b)


def test_hostsim_rejects_an_invalid_table():
    hs = _EpSim(_config(), 2)
    rows = np.tile(_abi.config_env_params(_config()), (2, 1))
    rows[1, _abi.EP_IMU_ACC_BIAS] = -0.5  # biases may be negative
    assert hs.set_env_params(rows) & 1 == 0
    for col, bad in ((_abi.EP_KD, -1.0), (_abi.EP_FRICTION + 2, np.nan), (_abi.EP_IMU_ACC_BIAS, np.inf),
                     (_abi.EP_MEAS_NOISE, -1e-3)):
        r = rows.copy()
        r[0, col] = bad
        assert hs.set_env_params(r) & 1
