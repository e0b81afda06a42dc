# SPDX-License-Identifier: Apache-2.0
"""Vectorised Upkie environments on the sm_90a kernels.

``B200VectorEnv`` is a ``gymnasium.vector.VectorEnv`` whose
``single_action_space`` / ``single_observation_space`` are identical to the
reference's single-robot environments:

- ``"servos"``   = ``UpkieServos``   (``upkie/envs/upkie_servos.py:20-344``)
- ``"gyropod"``  = ``UpkieGyropod``  (``upkie/envs/upkie_gyropod.py:20-392``)
- ``"pendulum"`` = ``UpkiePendulum`` (``upkie/envs/upkie_pendulum.py:20-142``)

with the reference's reset semantics (seeded NumPy sampling of the initial
state, ``upkie/envs/upkie_env.py:162-194``), ``reward == 0.0`` and
``truncated == False`` (``upkie_env.py:230-232``), fall termination for the
wheeled-inverted-pendulum wrappers (``upkie_gyropod.py:333-352``).

``max_episode_steps=T`` adds the time limit of Gymnasium's ``TimeLimit`` wrapper
per env inside the step kernel (``truncated`` once an env has run T steps since
its last reset), which the fused auto-reset honours.
"""

from typing import Any, Dict, Optional, Sequence, Tuple, Union

import numpy as np
import torch

from . import _abi
from .base_velocity import base_velocity_post
from .exceptions import UpkieException, UpkieRuntimeError
from .gym_compat import VectorEnv, batch_space, spaces
from .model import Model, default_model
from .robot_state import RobotState
from .sim import AUTORESET_DISABLED, AUTORESET_NEXT_STEP, AUTORESET_SAME_STEP, UpkieSim

ENV_TYPES = ("servos", "gyropod", "pendulum", "base_velocity")
_AUTORESET = {"disabled": AUTORESET_DISABLED, "next_step": AUTORESET_NEXT_STEP, "same_step": AUTORESET_SAME_STEP}


# ---- spaces (host-side, no GPU needed) ------------------------------------------------

def make_servo_spaces(model: Model, max_gain_scale: float = 5.0):
    """``UpkieServos.__create_servo_spaces`` (``upkie_servos.py:173-286``).

    Returns ``(action_space, observation_space, neutral_action, max_action,
    min_action)``.
    """
    if not (0.0 < max_gain_scale < 10.0):
        raise UpkieRuntimeError(f"Invalid value {max_gain_scale=}")
    action_space, servo_space = {}, {}
    neutral_action, max_action, min_action = {}, {}, {}
    f32 = np.float32

    def box(lo, hi):
        return spaces.Box(low=lo, high=hi, shape=(1,), dtype=f32)

    for joint in model.joints:
        lim = joint.limit
        action_space[joint.name] = spaces.Dict(
            {
                "position": box(lim.lower, lim.upper),
                "velocity": box(-lim.velocity, +lim.velocity),
                "feedforward_torque": box(-lim.effort, +lim.effort),
                "kp_scale": box(0.0, max_gain_scale),
                "kd_scale": box(0.0, max_gain_scale),
                "maximum_torque": box(0.0, lim.effort),
            }
        )
        servo_space[joint.name] = spaces.Dict(
            {
                "position": box(lim.lower, lim.upper),
                "velocity": box(-lim.velocity, +lim.velocity),
                "torque": box(-lim.effort, +lim.effort),
                "temperature": box(0.0, 100.0),
                "voltage": box(10.0, 44.0),  # moteus min 10 V, max 44 V
            }
        )
        neutral_action[joint.name] = {
            "position": np.nan,
            "velocity": 0.0,
            "feedforward_torque": 0.0,
            "kp_scale": 1.0,
            "kd_scale": 1.0,
            "maximum_torque": lim.effort,
        }
        max_action[joint.name] = {
            "position": lim.upper,
            "velocity": lim.velocity,
            "feedforward_torque": lim.effort,
            "kp_scale": max_gain_scale,
            "kd_scale": max_gain_scale,
            "maximum_torque": lim.effort,
        }
        min_action[joint.name] = {
            "position": lim.lower,
            "velocity": -lim.velocity,
            "feedforward_torque": -lim.effort,
            "kp_scale": 0.0,
            "kd_scale": 0.0,
            "maximum_torque": 0.0,
        }
    return spaces.Dict(action_space), spaces.Dict(servo_space), neutral_action, max_action, min_action


def make_gyropod_spaces(max_ground_velocity: float = 3.0, max_yaw_velocity: float = 1.0):
    """``UpkieGyropod.__init__`` spaces (``upkie_gyropod.py:118-160``)."""
    observation_limit = np.array(
        [float("inf"), np.pi, float("inf"), max_ground_velocity, 1000.0, max_yaw_velocity], dtype=np.float32
    )
    action_limit = np.array([max_ground_velocity, max_yaw_velocity], dtype=np.float32)
    obs = spaces.Box(-observation_limit, +observation_limit, shape=observation_limit.shape, dtype=observation_limit.dtype)
    act = spaces.Box(-action_limit, +action_limit, shape=action_limit.shape, dtype=action_limit.dtype)
    return act, obs


PENDULUM_OBS_INDICES = [1, 0, 4, 3]  # upkie_pendulum.py:17


def make_pendulum_spaces(max_ground_velocity: float = 3.0):
    """``UpkiePendulum.__init__`` spaces (``upkie_pendulum.py:87-102``)."""
    _, gyro_obs = make_gyropod_spaces(max_ground_velocity)
    obs_limit = gyro_obs.high[PENDULUM_OBS_INDICES]
    obs = spaces.Box(-obs_limit, +obs_limit, shape=obs_limit.shape, dtype=np.float32)
    action_limit = np.array([max_ground_velocity], dtype=np.float32)
    act = spaces.Box(-action_limit, +action_limit, shape=action_limit.shape, dtype=np.float32)
    return act, obs


def make_base_velocity_spaces(max_ground_velocity: float = 3.0, max_yaw_velocity: float = 1.0):
    """``UpkieBaseVelocity.__init__`` spaces (``upkie_base_velocity.py:96-115``)."""
    observation_limit = np.full(3, float("inf"), dtype=np.float32)
    action_limit = np.array([max_ground_velocity, max_yaw_velocity], dtype=np.float32)
    obs = spaces.Box(-observation_limit, +observation_limit, shape=observation_limit.shape, dtype=observation_limit.dtype)
    act = spaces.Box(-action_limit, +action_limit, shape=action_limit.shape, dtype=action_limit.dtype)
    return act, obs


def servo_action_dict_to_array(action: dict, neutral_action: dict, n: int) -> np.ndarray:
    """Batched dict action ``{joint: {key: array[N, 1]}}`` -> ``[N, 6, 6]``.
    Missing keys take the neutral action (``upkie_servos.py:326-331``)."""
    out = np.empty((n, 6, 6), dtype=np.float32)
    for j, name in enumerate(_abi.JOINT_NAMES):
        ja = action.get(name, {}) if isinstance(action, dict) else {}
        for k, key in enumerate(_abi.ACT_KEYS):
            if key in ja:
                out[:, j, k] = np.asarray(ja[key], dtype=np.float32).reshape(n)
            else:
                out[:, j, k] = neutral_action[name][key]
    return out


def servo_obs_array_to_dict(obs: np.ndarray) -> dict:
    """``[N, 6, 5]`` -> batched dict ``{joint: {key: array[N, 1] float32}}``
    (``UpkieServos.get_env_observation``, ``upkie_servos.py:288-306``)."""
    return {
        name: {key: obs[:, j, k : k + 1].astype(np.float32, copy=False) for k, key in enumerate(_abi.OBS_KEYS)}
        for j, name in enumerate(_abi.JOINT_NAMES)
    }


class SpineObservations:
    """Lazy ``info["spine_observation"]``: fetched from the device on first use.

    ``obs[i]`` returns the reference's nested dictionary for env ``i``
    (``pybullet_backend.py:325-331``); ``obs.array`` the flat ``[N, 62]`` array,
    ``obs.tensor`` the same rows as a CUDA tensor (no host copy).

    With an observation history (``B200VectorEnv(history=...)``), ``obs.history`` is the batched ``[N, K, C]`` CUDA
    tensor of ``UpkieSim.get_history`` and ``obs[i]`` has a ``"history"`` subtree in ``HistoryObserver``'s layout (the
    key path of each recorded value holds its ``K`` values, newest first), fetched and stale-checked like ``.tensor``.
    """

    _key = "info['spine_observation']"

    def __init__(self, sim: UpkieSim, history_layout: Optional[list] = None):
        self._sim = sim
        self._tensor = None
        self._array = None
        self._history_layout = history_layout  # [(key path, first column in the history, shape)], None = no history
        self._history = None
        self._history_array = None
        self._stamp = sim.launches  # step kernels launched so far: identifies the tick this object belongs to

    def _fetch(self) -> torch.Tensor:
        return self._sim.spine_obs()

    @property
    def tensor(self) -> torch.Tensor:
        if self._tensor is None:
            if self._sim.launches != self._stamp:
                # the simulator has moved on: fetching now would silently return a LATER tick's observation
                raise UpkieRuntimeError(
                    f"{self._key} is fetched lazily and the simulator has been stepped since this step: "
                    "read it (e.g. `.array`) before calling step() again")
            self._tensor = self._fetch()
        return self._tensor

    @property
    def array(self) -> np.ndarray:
        if self._array is None:
            self._array = self.tensor.cpu().numpy()
        return self._array

    def _check_stamp(self) -> None:
        if self._sim.launches != self._stamp:
            # the simulator has moved on: fetching now would silently return a LATER tick's history
            raise UpkieRuntimeError(
                f"{self._key} is fetched lazily and the simulator has been stepped since this step: "
                "read it (e.g. `.history`) before calling step() again")

    @property
    def history(self) -> torch.Tensor:
        """``[N, K, C]`` the observation history of every env (``UpkieSim.get_history``), newest entry first."""
        if self._history_layout is None:
            raise UpkieException(f"{self._key}: the env records no history (B200VectorEnv(history=...))")
        if self._history is None:
            self._check_stamp()
            self._history = self._sim.get_history()
        return self._history

    def __len__(self):
        return self._sim.n

    def __getitem__(self, i: int) -> dict:
        d = spine_row_to_dict(self.array[i])
        if self._history_layout is not None:
            if self._history_array is None:
                self._history_array = self.history.cpu().numpy()
            d["history"] = history_to_dict(self._history_layout, self._history_array[i])
        return d


class FinalSpineObservations(SpineObservations):
    """Lazy ``info["final_info"]["spine_observation"]`` of a same-step auto-reset step: the spine observation of the
    terminal step, row ``i`` for each env ``i`` that reset (``info["_final_info"]``), computed from the state the env
    stashed before its reset (``UpkieSim.final_spine_obs``). Same access as ``SpineObservations``; rows outside the
    mask are stale."""

    _key = "info['final_info']['spine_observation']"

    def __init__(self, sim: UpkieSim):
        super().__init__(sim)  # no history: the terminal step's history is not kept

    def _fetch(self) -> torch.Tensor:
        return self._sim.final_spine_obs()


def spine_row_to_dict(r: np.ndarray) -> dict:
    """Flat spine observation row -> the dictionary of
    ``PyBulletBackend.get_spine_observation``."""
    A = _abi
    return {
        "base_orientation": {
            "angular_velocity": [float(x) for x in r[A.SP_BASE_ANGVEL : A.SP_BASE_ANGVEL + 3]],
            "linear_velocity": [float(x) for x in r[A.SP_BASE_LINVEL : A.SP_BASE_LINVEL + 3]],
            "pitch": float(r[A.SP_PITCH]),
            "rotation_base_to_world": np.asarray(r[A.SP_ROT : A.SP_ROT + 9], dtype=float).reshape(3, 3).tolist(),
        },
        "floor_contact": {"contact": bool(r[A.SP_CONTACT] > 0.5)},
        "imu": {
            "orientation": [float(x) for x in r[A.SP_IMU_QUAT : A.SP_IMU_QUAT + 4]],
            "angular_velocity": [float(x) for x in r[A.SP_IMU_ANGVEL : A.SP_IMU_ANGVEL + 3]],
            "linear_acceleration": np.asarray(r[A.SP_IMU_LINACC : A.SP_IMU_LINACC + 3], dtype=float),
            "raw_linear_acceleration": [float(x) for x in r[A.SP_IMU_RAWACC : A.SP_IMU_RAWACC + 3]],
        },
        "servo": {
            name: {
                key: float(r[A.SP_SERVO + j * 5 + k]) for k, key in enumerate(A.OBS_KEYS)
            }
            for j, name in enumerate(A.JOINT_NAMES)
        },
        "wheel_odometry": {"position": float(r[A.SP_ODOM_POS]), "velocity": float(r[A.SP_ODOM_VEL])},
    }


# The spine observation's keys (spine_row_to_dict's table) as key path -> (first column, shape of the value): the
# history records these columns, a vector or matrix key all of its columns
def _history_keys() -> dict:
    A = _abi
    keys = {
        ("base_orientation", "angular_velocity"): (A.SP_BASE_ANGVEL, (3,)),
        ("base_orientation", "linear_velocity"): (A.SP_BASE_LINVEL, (3,)),
        ("base_orientation", "pitch"): (A.SP_PITCH, ()),
        ("base_orientation", "rotation_base_to_world"): (A.SP_ROT, (3, 3)),
        ("floor_contact", "contact"): (A.SP_CONTACT, ()),
        ("imu", "orientation"): (A.SP_IMU_QUAT, (4,)),
        ("imu", "angular_velocity"): (A.SP_IMU_ANGVEL, (3,)),
        ("imu", "linear_acceleration"): (A.SP_IMU_LINACC, (3,)),
        ("imu", "raw_linear_acceleration"): (A.SP_IMU_RAWACC, (3,)),
        ("wheel_odometry", "position"): (A.SP_ODOM_POS, ()),
        ("wheel_odometry", "velocity"): (A.SP_ODOM_VEL, ()),
    }
    for j, name in enumerate(A.JOINT_NAMES):
        for k, key in enumerate(A.OBS_KEYS):
            keys[("servo", name, key)] = (A.SP_SERVO + j * len(A.OBS_KEYS) + k, ())
    return keys


_CONSTANT_KEYS = ("temperature", "voltage")  # servo keys the simulation reports as constants


def history_spec(keys, size: int = 1, spine_mode: bool = False, joint_limits: int = 3,
                 body_contacts: bool = False) -> Optional[Tuple[list, int, list]]:
    """``(columns, size, layout)`` of an observation history from key paths of the spine observation dictionary,
    e.g. ``("imu", "angular_velocity")``, ``("base_orientation", "pitch")``, ``("servo", "left_wheel", "velocity")``
    (tuples, or strings with ``/`` between the keys). A vector key records its 3 (or 4) columns, the rotation matrix its
    9. ``layout`` lists ``(key path, first column in the history, shape)``. None for ``keys=None``. Raises on an unknown
    key, a constant servo key (temperature, voltage), more than ``MAX_HISTORY_CHANNELS`` columns, a size outside 1 ..
    ``MAX_HISTORY``, and the configurations the history does not run in, before any device is touched."""
    if keys is None:
        return None
    if isinstance(keys, (str, tuple)):
        keys = [keys]
    table = _history_keys()
    columns, layout = [], []
    for key in keys:
        path = tuple(key.strip("/").split("/")) if isinstance(key, str) else tuple(key)
        if len(path) == 3 and path[0] == "servo" and path[2] in _CONSTANT_KEYS:
            raise UpkieException(f"history: {'/'.join(path)} is a constant of the simulation, not a measurement")
        if path not in table:
            raise UpkieException(f"history: unknown key {'/'.join(map(str, path))} of the spine observation")
        col, shape = table[path]
        layout.append((path, len(columns), shape))
        columns.extend(range(col, col + int(np.prod(shape, dtype=int))))
    if not 1 <= len(columns) <= _abi.MAX_HISTORY_CHANNELS:
        raise UpkieException(f"history: 1 to {_abi.MAX_HISTORY_CHANNELS} columns, the keys give {len(columns)}")
    if int(size) != size or not 1 <= size <= _abi.MAX_HISTORY:
        raise UpkieException(f"history_size must be an integer in [1, {_abi.MAX_HISTORY}], got {size!r}")
    if spine_mode:
        raise UpkieException("history: spine_mode reports the spine's lagged replies, which the history does not record")
    if not joint_limits:
        raise UpkieException("history: needs joint_limits (the history runs in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("history: body_contacts has no observation-history kernels")
    return columns, int(size), layout


def history_to_dict(layout: list, h: np.ndarray) -> dict:
    """One env's history ``h[K, C]`` as the ``observation["history"]`` subtree of the reference's HistoryObserver: each
    key path holds the list of its ``K`` values, newest first."""
    out: dict = {}
    for path, c0, shape in layout:
        node = out
        for key in path[:-1]:
            node = node.setdefault(key, {})
        size = int(np.prod(shape, dtype=int))
        vals = h[:, c0 : c0 + size].astype(float)
        if path == ("floor_contact", "contact"):
            node[path[-1]] = [bool(v > 0.5) for v in vals[:, 0]]
        elif shape == ():
            node[path[-1]] = [float(v) for v in vals[:, 0]]
        else:
            node[path[-1]] = [v.reshape(shape).tolist() for v in vals]
    return out


def _check_max_episode_steps(value) -> int:
    if value is None:
        return 0
    if int(value) != value or value < 0 or value > 0x7FFFFFFF:
        raise UpkieException(f"max_episode_steps must be an integer in [0, 2**31), got {value!r} (0 = no time limit)")
    return int(value)


def make_config(
    frequency: float = 200.0,
    nb_substeps: Optional[int] = None,
    torque_control_kp: float = 20.0,
    torque_control_kd: float = 1.0,
    joint_properties: Optional[dict] = None,
    max_gain_scale: float = 5.0,
    fall_pitch: float = 1.0,
    leg_gain_scale: float = 1.0,
    max_ground_velocity: float = 3.0,
    max_yaw_velocity: float = 1.0,
    init_state: Optional[RobotState] = None,
    noise_seed: int = 0,
    joint_limits: Union[bool, int] = True,
    spine_mode: bool = False,
    body_contacts: bool = False,
    max_episode_steps: int = 0,
) -> _abi.UpkieSimConfig:
    """Split of the keyword arguments the reference's factories forward to the
    backend, the servo env and the wrappers (``upkie/envs/entry_points.py:41-61,99-109``).
    ``max_episode_steps``: per-env time limit in agent steps, 0 = none (include/upkie_b200.h)."""
    if frequency is None:
        raise UpkieException("This environment needs a loop frequency")
    max_episode_steps = _check_max_episode_steps(max_episode_steps)
    cfg = _abi.default_sim_config(frequency)
    if nb_substeps is not None:
        cfg.nb_substeps = int(nb_substeps)
    if cfg.nb_substeps < 1:
        cfg.nb_substeps = 1
    cfg.torque_control_kp = torque_control_kp
    cfg.torque_control_kd = torque_control_kd
    for j, name in enumerate(_abi.JOINT_NAMES):
        props = (joint_properties or {}).get(name)
        if props is not None:
            cfg.joint_friction[j] = float(getattr(props, "friction", 0.0))
            cfg.torque_control_noise[j] = float(getattr(props, "torque_control_noise", 0.0))
            cfg.torque_measurement_noise[j] = float(getattr(props, "torque_measurement_noise", 0.0))
    cfg.noise_seed = int(noise_seed) & 0xFFFFFFFFFFFFFFFF
    # Bullet's joint-limit constraint rows on hips and knees (include/upkie_b200.h: joint_limits): on, as in the
    # multibody PyBullet's importer builds (pybullet_backend.py:121). True -> 3 (the packed ten-row solver for the warps
    # that hold a robot on a bound); 2 = ten-row solver for every warp; False / 0 = no limit rows (round-1 behaviour)
    cfg.joint_limits = 3 if joint_limits is True else int(joint_limits)
    # timing of the C++ Bullet spine in simulate() mode instead of PyBulletBackend's (include/upkie_b200.h: spine_mode)
    cfg.spine_mode = 1 if spine_mode else 0
    # body-ground contacts (include/upkie_b200.h: body_contacts): the collision shapes of the model's links other than
    # the tires hold contact rows against the floor, as they do in Bullet; needs the joint-limit kernels
    cfg.body_contacts = 1 if (body_contacts and cfg.joint_limits) else 0
    cfg.max_gain_scale = max_gain_scale
    cfg.fall_pitch = fall_pitch
    cfg.leg_gain_scale = leg_gain_scale
    cfg.max_ground_velocity = max_ground_velocity
    cfg.max_yaw_velocity = max_yaw_velocity
    cfg.max_episode_steps = max_episode_steps
    if init_state is not None:
        init_state.apply_to_config(cfg)
    return cfg


_JOINT_PROPERTY_COLUMNS = (
    ("friction", _abi.EP_FRICTION),
    ("torque_control_noise", _abi.EP_CTRL_NOISE),
    ("torque_measurement_noise", _abi.EP_MEAS_NOISE),
)


def _per_env(value) -> bool:
    return np.ndim(value) != 0


def needs_env_params(torque_control_kp=None, torque_control_kd=None, joint_properties=None) -> bool:
    """Whether these ``B200VectorEnv`` arguments differ between envs: ``[N]`` arrays, ``JointProperties`` with
    array fields, or a sequence of per-env ``joint_properties`` dicts. All-scalar arguments fit in the config."""
    if _per_env(torque_control_kp) or _per_env(torque_control_kd):
        return True
    if joint_properties is None:
        return False
    if not isinstance(joint_properties, dict):
        return True
    return any(_per_env(getattr(props, f, 0.0)) for props in joint_properties.values() for f, _ in _JOINT_PROPERTY_COLUMNS)


def env_params_table(num_envs: int, base: np.ndarray, torque_control_kp=None, torque_control_kd=None,
                     joint_properties=None) -> np.ndarray:
    """Per-env parameter table ``[N, EP_DIM]`` float32 (``UpkieSim.set_env_params``) from the reference's constructor
    arguments (``PyBulletBackend(torque_control_kp, torque_control_kd, joint_properties)``, ``pybullet_backend.py:55-65``).
    ``base``: a configuration's row (``_abi.config_env_params``) or a table ``[N, EP_DIM]``; it fills every column the
    arguments do not give (None = not given). Gains take a float or an ``[N]`` array. ``joint_properties`` takes
    ``{joint: JointProperties}`` whose fields are floats or ``[N]`` arrays, or a sequence of N such dicts, one per env.
    Raises ``UpkieException`` on a wrong length, a non-finite or a negative value."""
    n = int(num_envs)
    table = np.empty((n, _abi.EP_DIM), dtype=np.float32)  # C order, as the C ABI reads it
    table[:] = np.asarray(base, dtype=np.float32)

    def column(value, name):
        v = np.asarray(value, dtype=np.float64)
        if v.ndim > 1 or (v.ndim == 1 and v.shape[0] != n):
            raise UpkieException(f"{name}: expected a float or an array of {n} values, got shape {v.shape}")
        if not np.all(np.isfinite(v)) or np.any(v < 0.0):
            raise UpkieException(f"{name}: values must be finite and >= 0")
        return np.broadcast_to(v, (n,)).astype(np.float32)

    if torque_control_kp is not None:
        table[:, _abi.EP_KP] = column(torque_control_kp, "torque_control_kp")
    if torque_control_kd is not None:
        table[:, _abi.EP_KD] = column(torque_control_kd, "torque_control_kd")
    if joint_properties is None:
        return table
    if isinstance(joint_properties, dict):
        per_joint = [(None, joint_properties)]
    else:
        if len(joint_properties) != n:
            raise UpkieException(f"joint_properties: expected one dict per env ({n}), got {len(joint_properties)}")
        per_joint = list(enumerate(joint_properties))
    for env, props_of in per_joint:
        for j, name in enumerate(_abi.JOINT_NAMES):
            props = (props_of or {}).get(name)
            if props is None:
                continue
            for field, col in _JOINT_PROPERTY_COLUMNS:
                value = getattr(props, field, 0.0)
                if env is None:
                    table[:, col + j] = column(value, f"joint_properties[{name!r}].{field}")
                elif _per_env(value):
                    raise UpkieException(f"joint_properties[{env}][{name!r}].{field}: a per-env dict takes floats")
                else:
                    table[env, col + j] = column(value, f"joint_properties[{env}][{name!r}].{field}")[0]
    return table


_IMU_RANGE_COLUMNS = {
    "accelerometer_bias": (_abi.EP_IMU_ACC_BIAS, 3),
    "accelerometer_noise": (_abi.EP_IMU_ACC_NOISE, 1),
    "gyroscope_bias": (_abi.EP_IMU_GYRO_BIAS, 3),
    "gyroscope_noise": (_abi.EP_IMU_GYRO_NOISE, 1),
}


def reset_randomization_spec(spec: Optional[dict]) -> Optional[_abi.UpkieResetRandomization]:
    """``UpkieResetRandomization`` (``UpkieSim.set_reset_randomization``) from a dict in the argument forms of the
    constructor: ``inertia_variation=v`` (``[-v, v]`` on the six bodies, as ``randomize_inertias``),
    ``floor_friction=(lo, hi)``, ``torque_control_kp`` / ``torque_control_kd=(lo, hi)``,
    ``joint_properties={joint: {"friction" | "torque_control_noise" | "torque_measurement_noise": (lo, hi)}}`` and
    ``imu_uncertainty={"accelerometer_bias" | "accelerometer_noise" | "gyroscope_bias" | "gyroscope_noise": (lo, hi)}``
    whose bias bounds are floats or per-axis triples. Every reset of an env draws the given columns uniformly from their
    ranges; the others keep their values. Raises ``UpkieException`` on an unknown key or joint, a bound that is not
    finite, ``lo > hi``, a negative low bound on a gain, friction or noise level, or an inertia bound <= -1."""
    if spec is None:
        return None
    out = _abi.UpkieResetRandomization()
    out.columns = 0

    def put(col, lo, hi, name, min_low=None):
        lo, hi = float(lo), float(hi)
        if not (np.isfinite(lo) and np.isfinite(hi)) or lo > hi:
            raise UpkieException(f"{name}: expected finite bounds with low <= high, got ({lo}, {hi})")
        if min_low is not None and not lo >= min_low:
            raise UpkieException(f"{name}: low bound must be >= {min_low}, got {lo}")
        out.columns |= 1 << col
        out.low[col], out.high[col] = lo, hi

    def pair(value, name):
        try:
            lo, hi = value
        except (TypeError, ValueError):
            raise UpkieException(f"{name}: expected a (low, high) pair, got {value!r}") from None
        return lo, hi

    known = {"inertia_variation", "floor_friction", "torque_control_kp", "torque_control_kd", "joint_properties",
             "imu_uncertainty"}
    unknown = set(spec) - known
    if unknown:
        raise UpkieException(f"reset_randomization: unknown keys {sorted(unknown)} (known: {sorted(known)})")
    if spec.get("inertia_variation") is not None:
        v = float(spec["inertia_variation"])
        if not (np.isfinite(v) and 0.0 <= v < 1.0):
            raise UpkieException(f"inertia_variation: expected 0 <= v < 1, got {v}")
        for b in range(6):
            put(_abi.RR_INERTIA + b, -v, v, "inertia_variation")
    if spec.get("floor_friction") is not None:
        put(_abi.RR_FRICTION, *pair(spec["floor_friction"], "floor_friction"), "floor_friction", 0.0)
    for name, col in (("torque_control_kp", _abi.EP_KP), ("torque_control_kd", _abi.EP_KD)):
        if spec.get(name) is not None:
            put(col, *pair(spec[name], name), name, 0.0)
    fields = dict(_JOINT_PROPERTY_COLUMNS)
    for joint, props in (spec.get("joint_properties") or {}).items():
        if joint not in _abi.JOINT_NAMES:
            raise UpkieException(f"joint_properties: unknown joint {joint!r} (joints: {_abi.JOINT_NAMES})")
        for field, value in props.items():
            if field not in fields:
                raise UpkieException(f"joint_properties[{joint!r}]: unknown field {field!r} (fields: {tuple(fields)})")
            name = f"joint_properties[{joint!r}].{field}"
            put(fields[field] + _abi.JOINT_NAMES.index(joint), *pair(value, name), name, 0.0)
    for key, value in (spec.get("imu_uncertainty") or {}).items():
        if key not in _IMU_RANGE_COLUMNS:
            raise UpkieException(f"imu_uncertainty: unknown key {key!r} (keys: {tuple(_IMU_RANGE_COLUMNS)})")
        col, dim = _IMU_RANGE_COLUMNS[key]
        lo, hi = pair(value, f"imu_uncertainty[{key!r}]")
        lo = np.broadcast_to(np.asarray(lo, dtype=np.float64), (dim,))
        hi = np.broadcast_to(np.asarray(hi, dtype=np.float64), (dim,))
        for k in range(dim):
            put(col + k, lo[k], hi[k], f"imu_uncertainty[{key!r}]", None if dim == 3 else 0.0)
    return out


def push_randomization_spec(spec: Optional[dict], model: Model, dt: float) -> Optional[_abi.UpkiePushRandomization]:
    """``UpkiePushRandomization`` (``UpkieSim.set_push_randomization``) from a dict ``{"link": name, "interval": (lo,
    hi), "duration": (lo, hi), "force": ((fx, fy, fz) low, (fx, fy, fz) high)}``: after every reset, an env waits a gap
    drawn from ``interval`` seconds, is pushed for a time drawn from ``duration`` seconds by a world-frame force drawn
    from ``force`` newtons (bounds: floats or per-axis triples) on ``link``, then draws the next push. Times are rounded
    to the nearest step of ``dt`` (halves up). A link maps to the body it is lumped into, as in
    ``Model.external_force_rows``. Raises ``UpkieException`` on an unknown key or link, a bound that is not finite,
    ``lo > hi``, a negative time, a duration that rounds to 0 steps, or more than ``_abi.PUSH_MAX_STEPS`` steps."""
    if spec is None:
        return None
    known = {"link", "interval", "duration", "force"}
    unknown = set(spec) - known
    if unknown:
        raise UpkieException(f"push_randomization: unknown keys {sorted(unknown)} (known: {sorted(known)})")
    missing = known - set(spec)
    if missing:
        raise UpkieException(f"push_randomization: missing keys {sorted(missing)}")
    link = spec["link"]
    if not isinstance(link, str) or link not in model.link_body:
        raise UpkieException(f"push_randomization: unknown link {link!r} (links: {sorted(model.link_body)})")

    def pair(value, name):
        try:
            lo, hi = value
        except (TypeError, ValueError):
            raise UpkieException(f"push_randomization[{name!r}]: expected a (low, high) pair, got {value!r}") from None
        return lo, hi

    def steps(name):
        lo, hi = (float(x) for x in pair(spec[name], name))
        if not (np.isfinite(lo) and np.isfinite(hi)) or not 0.0 <= lo <= hi:
            raise UpkieException(f"push_randomization[{name!r}]: expected finite seconds 0 <= low <= high, got "
                                 f"({lo}, {hi})")
        lo_s, hi_s = (int(np.floor(x / dt + 0.5)) for x in (lo, hi))
        if hi_s > _abi.PUSH_MAX_STEPS:
            raise UpkieException(f"push_randomization[{name!r}]: more than {_abi.PUSH_MAX_STEPS} steps")
        return lo_s, hi_s

    out = _abi.UpkiePushRandomization()
    out.body = int(model.link_body[link])
    out.gap_low, out.gap_high = steps("interval")
    out.duration_low, out.duration_high = steps("duration")
    if out.duration_low == 0:
        raise UpkieException(f"push_randomization['duration']: the low bound rounds to 0 steps of {dt} s")
    lo, hi = pair(spec["force"], "force")
    try:
        lo = np.broadcast_to(np.asarray(lo, dtype=np.float64), (3,))
        hi = np.broadcast_to(np.asarray(hi, dtype=np.float64), (3,))
    except ValueError:
        raise UpkieException(f"push_randomization['force']: expected floats or (fx, fy, fz) bounds") from None
    with np.errstate(over="ignore"):
        finite = np.all(np.isfinite(lo.astype(np.float32))) and np.all(np.isfinite(hi.astype(np.float32)))
    if not (finite and np.all(lo <= hi)):
        raise UpkieException(f"push_randomization['force']: expected finite bounds with low <= high, got ({lo}, {hi})")
    for a in range(3):
        out.force_low[a], out.force_high[a] = lo[a], hi[a]
    return out


def _check_max_delay_ticks(max_ticks) -> int:
    """``max_ticks`` of a delay as an int in ``1 .. MAX_DELAY_TICKS``, or ``UpkieException``"""
    if isinstance(max_ticks, (bool, np.bool_)) or not isinstance(max_ticks, (int, np.integer)):
        raise UpkieException(f"max_ticks: expected an integer, got {max_ticks!r}")
    if not 1 <= int(max_ticks) <= _abi.MAX_DELAY_TICKS:
        raise UpkieException(f"max_ticks: expected 1 <= max_ticks <= {_abi.MAX_DELAY_TICKS}, got {max_ticks}")
    return int(max_ticks)


def action_delay_spec(delay, dt: float, nb_substeps: int, spine_mode: bool = False,
                      joint_limits: Union[bool, int] = True, max_ticks: int = 1) -> Optional[Tuple[int, int]]:
    """``(substeps_low, substeps_high)`` (``UpkieSim.set_action_delay``) from an action delay in seconds: a float, or a
    ``(low, high)`` pair from which every reset draws an env's delay. Rounded to the nearest substep of ``dt /
    nb_substeps`` (halves up). Raises ``UpkieException`` on a negative or non-finite bound, ``low > high``, a delay
    of more than ``max_ticks`` ticks (``max_ticks * nb_substeps`` substeps; ``max_ticks`` from 1 to
    ``MAX_DELAY_TICKS``, the history the delay keeps), ``spine_mode`` (which models the spine's own lag) and no joint
    limits (the delay runs in the kernels with joint-limit rows)."""
    max_ticks = _check_max_delay_ticks(max_ticks)
    if delay is None:
        return None
    if isinstance(delay, (int, float, np.integer, np.floating)):
        lo, hi = delay, delay
    else:
        try:
            lo, hi = delay
        except (TypeError, ValueError):
            raise UpkieException(f"action_delay: expected seconds or a (low, high) pair, got {delay!r}") from None
    try:
        lo, hi = float(lo), float(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"action_delay: expected seconds, got ({lo!r}, {hi!r})") from None
    if not (np.isfinite(lo) and np.isfinite(hi)) or not 0.0 <= lo <= hi:
        raise UpkieException(f"action_delay: expected finite seconds 0 <= low <= high, got ({lo}, {hi})")
    if spine_mode:
        raise UpkieException("action_delay: spine_mode models the spine's own lag; the delay is not available there")
    if not joint_limits:
        raise UpkieException("action_delay: needs joint_limits (the delay runs in the kernels with joint-limit rows)")
    substep = dt / int(nb_substeps)
    lo_s, hi_s = (int(np.floor(x / substep + 0.5)) for x in (lo, hi))
    if max_ticks == 1 and hi_s > int(nb_substeps):
        raise UpkieException(f"action_delay: {hi} s is more than one tick ({nb_substeps} substeps of {substep} s)")
    if hi_s > max_ticks * int(nb_substeps):
        raise UpkieException(f"action_delay: {hi} s is more than max_ticks = {max_ticks} ticks ({nb_substeps} substeps "
                             f"of {substep} s each)")
    return lo_s, hi_s


def observation_delay_spec(delay, dt: float, nb_substeps: int, spine_mode: bool = False,
                           joint_limits: Union[bool, int] = True,
                           body_contacts: Union[bool, int] = False, max_ticks: int = 1) -> Optional[Tuple[int, int]]:
    """``(substeps_low, substeps_high)`` (``UpkieSim.set_observation_delay``) from an observation delay in seconds: a
    float, or a ``(low, high)`` pair from which every reset draws an env's delay. Rounded to the nearest substep of
    ``dt / nb_substeps`` (halves up). Raises ``UpkieException`` on a negative or non-finite bound, ``low > high``, a
    delay of more than ``max_ticks`` ticks (``max_ticks * nb_substeps`` substeps; ``max_ticks`` from 1 to
    ``MAX_DELAY_TICKS``, the history the delay keeps), ``spine_mode`` (which models the spine's own lag), no joint
    limits (the delay runs in the kernels with joint-limit rows) and ``body_contacts`` (no such kernels)."""
    max_ticks = _check_max_delay_ticks(max_ticks)
    if delay is None:
        return None
    if isinstance(delay, (int, float, np.integer, np.floating)):
        lo, hi = delay, delay
    else:
        try:
            lo, hi = delay
        except (TypeError, ValueError):
            raise UpkieException(f"observation_delay: expected seconds or a (low, high) pair, got {delay!r}") from None
    try:
        lo, hi = float(lo), float(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"observation_delay: expected seconds, got ({lo!r}, {hi!r})") from None
    if not (np.isfinite(lo) and np.isfinite(hi)) or not 0.0 <= lo <= hi:
        raise UpkieException(f"observation_delay: expected finite seconds 0 <= low <= high, got ({lo}, {hi})")
    if spine_mode:
        raise UpkieException("observation_delay: spine_mode models the spine's own lag; the delay is not available "
                             "there")
    if not joint_limits:
        raise UpkieException("observation_delay: needs joint_limits (the delay runs in the kernels with joint-limit "
                             "rows)")
    if body_contacts:
        raise UpkieException("observation_delay: body_contacts has no observation-delay kernels")
    substep = dt / int(nb_substeps)
    lo_s, hi_s = (int(np.floor(x / substep + 0.5)) for x in (lo, hi))
    if max_ticks == 1 and hi_s > int(nb_substeps):
        raise UpkieException(f"observation_delay: {hi} s is more than one tick ({nb_substeps} substeps of {substep} s)")
    if hi_s > max_ticks * int(nb_substeps):
        raise UpkieException(f"observation_delay: {hi} s is more than max_ticks = {max_ticks} ticks ({nb_substeps} substeps "
                             f"of {substep} s each)")
    return lo_s, hi_s


def servo_dropout_spec(prob, joints=None, spine_mode: bool = False, joint_limits: Union[bool, int] = True,
                       body_contacts: Union[bool, int] = False) -> Optional[_abi.UpkieServoDropout]:
    """``UpkieServoDropout`` (``UpkieSim.set_servo_dropout``) from a per-cycle reply loss probability: a float, or a
    ``(low, high)`` pair from which every reset draws an env's probability, and the names of the servos that may lose
    replies (``joints``, ``JOINT_NAMES``; None: all six). Raises ``UpkieException`` on a bound outside [0, 1] or not a
    number, ``low > high``, an unknown or empty joint list, ``spine_mode`` (whose spine reports its own replies), no
    joint limits and ``body_contacts`` (the dropouts run in the kernels of the observation delay)."""
    if prob is None:
        return None
    if isinstance(prob, (int, float, np.integer, np.floating)):
        lo, hi = prob, prob
    else:
        try:
            lo, hi = prob
        except (TypeError, ValueError):
            raise UpkieException(f"servo_dropout: expected a probability or a (low, high) pair, got {prob!r}") from None
    try:
        lo, hi = float(lo), float(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"servo_dropout: expected probabilities, got ({lo!r}, {hi!r})") from None
    if not 0.0 <= lo <= hi <= 1.0:
        raise UpkieException(f"servo_dropout: expected probabilities 0 <= low <= high <= 1, got ({lo}, {hi})")
    names = _abi.JOINT_NAMES if joints is None else list(joints)
    unknown = [j for j in names if j not in _abi.JOINT_NAMES]
    if unknown:
        raise UpkieException(f"servo_dropout_joints: unknown joint(s) {unknown}, expected names of {_abi.JOINT_NAMES}")
    if not names:
        raise UpkieException("servo_dropout_joints: at least one joint")
    if spine_mode:
        raise UpkieException("servo_dropout: spine_mode reports the spine's own servo replies; the dropouts are not "
                             "available there")
    if not joint_limits:
        raise UpkieException("servo_dropout: needs joint_limits (the dropouts run in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("servo_dropout: body_contacts has no servo-dropout kernels")
    mask = 0
    for j in names:
        mask |= 1 << _abi.JOINT_NAMES.index(j)
    return _abi.UpkieServoDropout(lo, hi, mask, 0)


_IMU_MISALIGNMENT_MAX = np.float32(np.pi / 4)  # the largest |bound| (the C check compares float32 values)


def imu_misalignment_spec(misalignment, spine_mode: bool = False, joint_limits: Union[bool, int] = True,
                          body_contacts: Union[bool, int] = False) -> Optional[_abi.UpkieImuMisalignment]:
    """``UpkieImuMisalignment`` (``UpkieSim.set_imu_misalignment``) from a dict with any of the keys ``roll``,
    ``pitch`` and ``yaw`` (radians), each a fixed angle or a ``(low, high)`` range every reset draws the env's angle
    from; a missing key is 0. Raises ``UpkieException`` on an unknown key, a bound that is not a finite number, ``low >
    high``, ``|bound| > pi/4`` (a misalignment, not a remount), ``spine_mode`` (whose spine models its own IMU), no
    joint limits and ``body_contacts`` (the misalignment runs in the kernels of the observation delay)."""
    if misalignment is None:
        return None
    if not isinstance(misalignment, dict):
        raise UpkieException(f"imu_misalignment: expected a dict of roll / pitch / yaw ranges, got {misalignment!r}")
    unknown = sorted(set(misalignment) - {"roll", "pitch", "yaw"})
    if unknown:
        raise UpkieException(f"imu_misalignment: unknown key(s) {unknown}, expected roll, pitch and yaw")
    bounds = []
    for key in ("roll", "pitch", "yaw"):
        r = misalignment.get(key, 0.0)
        if isinstance(r, (int, float, np.integer, np.floating)):
            lo, hi = r, r
        else:
            try:
                lo, hi = r
            except (TypeError, ValueError):
                raise UpkieException(f"imu_misalignment: {key}: expected an angle or a (low, high) pair, got {r!r}") \
                    from None
        try:
            lo, hi = np.float32(lo), np.float32(hi)
        except (TypeError, ValueError):
            raise UpkieException(f"imu_misalignment: {key}: expected angles, got ({lo!r}, {hi!r})") from None
        if not (np.isfinite(lo) and np.isfinite(hi)) or max(abs(lo), abs(hi)) > _IMU_MISALIGNMENT_MAX:
            raise UpkieException(f"imu_misalignment: {key}: expected finite angles within [-pi/4, pi/4] radians, got "
                                 f"({lo}, {hi})")
        if lo > hi:
            raise UpkieException(f"imu_misalignment: {key}: expected low <= high, got ({lo}, {hi})")
        bounds += [float(lo), float(hi)]
    if spine_mode:
        raise UpkieException("imu_misalignment: spine_mode models its spine's own IMU; the misalignment is not "
                             "available there")
    if not joint_limits:
        raise UpkieException("imu_misalignment: needs joint_limits (the misalignment runs in the kernels with "
                             "joint-limit rows)")
    if body_contacts:
        raise UpkieException("imu_misalignment: body_contacts has no IMU-misalignment kernels")
    return _abi.UpkieImuMisalignment(*bounds)


def attitude_filter_spec(attitude_filter, spine_mode: bool = False, joint_limits: Union[bool, int] = True,
                         body_contacts: Union[bool, int] = False,
                         dt: Optional[float] = None, nb_substeps: Optional[int] = None,
                         obs_delay_ticks: int = 1) -> Optional[_abi.UpkieAttitudeFilter]:
    """``UpkieAttitudeFilter`` (``UpkieSim.set_attitude_filter``) from a dict with keys ``kp`` (1/s, required),
    ``ki`` (1/s^2), ``roll`` and ``pitch`` (rad, the initial estimate error about the base axes), each a fixed value
    or a ``(low, high)`` range every reset draws the env's value from; a missing optional key is 0. Raises
    ``UpkieException`` on an unknown key, a bound that is not a finite number, ``low > high``, ``kp < 0`` or
    ``kp_high * dt / nb_substeps > 0.5`` (when ``dt`` and ``nb_substeps`` are given), ``ki < 0`` or ``ki > 10``,
    ``|roll|`` or ``|pitch| > pi/4``, ``spine_mode`` (whose spine models its own IMU), no joint limits,
    ``body_contacts`` (the filter runs in the kernels of the observation delay) and an observation delay of more than
    one tick."""
    if attitude_filter is None:
        return None
    if not isinstance(attitude_filter, dict) or "kp" not in attitude_filter:
        raise UpkieException(f"attitude_filter: expected a dict with keys kp, ki, roll and pitch, got "
                             f"{attitude_filter!r}")
    unknown = sorted(set(attitude_filter) - {"kp", "ki", "roll", "pitch"})
    if unknown:
        raise UpkieException(f"attitude_filter: unknown key(s) {unknown}, expected kp, ki, roll and pitch")
    bounds = {}
    for key in ("kp", "ki", "roll", "pitch"):
        r = attitude_filter.get(key, 0.0)
        if isinstance(r, (int, float, np.integer, np.floating)):
            lo, hi = r, r
        else:
            try:
                lo, hi = r
            except (TypeError, ValueError):
                raise UpkieException(f"attitude_filter: {key}: expected a value or a (low, high) pair, got {r!r}") \
                    from None
        try:
            lo, hi = np.float32(lo), np.float32(hi)
        except (TypeError, ValueError):
            raise UpkieException(f"attitude_filter: {key}: expected numbers, got ({lo!r}, {hi!r})") from None
        if not (np.isfinite(lo) and np.isfinite(hi)):
            raise UpkieException(f"attitude_filter: {key}: expected finite bounds, got ({lo}, {hi})")
        if lo > hi:
            raise UpkieException(f"attitude_filter: {key}: expected low <= high, got ({lo}, {hi})")
        bounds[key] = (lo, hi)
    if bounds["kp"][0] < 0:
        raise UpkieException(f"attitude_filter: kp: expected gains >= 0, got {bounds['kp']}")
    if dt is not None and nb_substeps is not None:
        h = np.float32(np.float64(dt) / np.float64(nb_substeps))
        if float(bounds["kp"][1]) * float(h) > _abi.ATTITUDE_FILTER_MAX_KP_H:
            raise UpkieException(f"attitude_filter: kp: kp_high * (dt / nb_substeps) must stay <= "
                                 f"{_abi.ATTITUDE_FILTER_MAX_KP_H}, got {bounds['kp'][1]} * {h}")
    if bounds["ki"][0] < 0 or bounds["ki"][1] > np.float32(_abi.ATTITUDE_FILTER_MAX_KI):
        raise UpkieException(f"attitude_filter: ki: expected 0 <= ki <= {_abi.ATTITUDE_FILTER_MAX_KI}, got "
                             f"{bounds['ki']}")
    for key in ("roll", "pitch"):
        if max(abs(bounds[key][0]), abs(bounds[key][1])) > np.float32(_abi.ATTITUDE_FILTER_MAX_ERROR):
            raise UpkieException(f"attitude_filter: {key}: expected errors within [-pi/4, pi/4] radians, got "
                                 f"{bounds[key]}")
    if spine_mode:
        raise UpkieException("attitude_filter: spine_mode models its spine's own IMU; the filter is not available there")
    if not joint_limits:
        raise UpkieException("attitude_filter: needs joint_limits (the filter runs in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("attitude_filter: body_contacts has no attitude-filter kernels")
    if obs_delay_ticks > 1:
        raise UpkieException("attitude_filter: not with an observation delay of more than one tick (its report would "
                             "need a ring of estimates)")
    return _abi.UpkieAttitudeFilter(*(float(v) for key in ("kp", "ki", "roll", "pitch") for v in bounds[key]))


def _set_attitude_filter(sim, spec: Optional[_abi.UpkieAttitudeFilter]) -> None:
    if spec is None:
        sim.set_attitude_filter(None)
    else:
        sim.set_attitude_filter((spec.kp_low, spec.kp_high), (spec.ki_low, spec.ki_high),
                                (spec.roll_low, spec.roll_high), (spec.pitch_low, spec.pitch_high))


_ENCODER_OFFSET_MAX = np.float32(0.5)  # the largest |bound|, radians (the C check compares float32 values)


def encoder_offset_spec(offset, joints=None, spine_mode: bool = False, joint_limits: Union[bool, int] = True,
                        body_contacts: Union[bool, int] = False) -> Optional[_abi.UpkieEncoderOffset]:
    """``UpkieEncoderOffset`` (``UpkieSim.set_encoder_offset``) from a servo encoder zero offset in radians: a bound
    ``b`` (the range ``(-b, b)``), or a ``(low, high)`` pair from which every reset draws each joint's offset, and the
    names of the joints that have one (``joints``, ``JOINT_NAMES``; None: the four hip and knee joints, which are zeroed
    by hand on the robot). Raises ``UpkieException`` on a bound that is not a finite number, ``low > high``, ``|bound| >
    0.5`` (a calibration error, not a remount), an unknown or empty joint list, ``spine_mode`` (whose spine reports its
    own servos), no joint limits and ``body_contacts`` (the offsets run in the kernels of the observation delay)."""
    if offset is None:
        return None
    if isinstance(offset, (int, float, np.integer, np.floating)):
        lo, hi = -abs(offset), abs(offset)
    else:
        try:
            lo, hi = offset
        except (TypeError, ValueError):
            raise UpkieException(f"encoder_offset: expected a bound or a (low, high) pair, got {offset!r}") from None
    try:
        lo, hi = np.float32(lo), np.float32(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"encoder_offset: expected angles, got ({lo!r}, {hi!r})") from None
    if not (np.isfinite(lo) and np.isfinite(hi)) or max(abs(lo), abs(hi)) > _ENCODER_OFFSET_MAX:
        raise UpkieException(f"encoder_offset: expected finite angles within [-0.5, 0.5] radians, got ({lo}, {hi})")
    if lo > hi:
        raise UpkieException(f"encoder_offset: expected low <= high, got ({lo}, {hi})")
    names = list(_abi.ENCODER_OFFSET_DEFAULT_JOINTS) if joints is None else list(joints)
    unknown = [j for j in names if j not in _abi.JOINT_NAMES]
    if unknown:
        raise UpkieException(f"encoder_offset_joints: unknown joint(s) {unknown}, expected names of {_abi.JOINT_NAMES}")
    if not names:
        raise UpkieException("encoder_offset_joints: at least one joint")
    if spine_mode:
        raise UpkieException("encoder_offset: spine_mode reports the spine's own servos; the offsets are not available "
                             "there")
    if not joint_limits:
        raise UpkieException("encoder_offset: needs joint_limits (the offsets run in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("encoder_offset: body_contacts has no encoder-offset kernels")
    mask = 0
    for j in names:
        mask |= 1 << _abi.JOINT_NAMES.index(j)
    return _abi.UpkieEncoderOffset(float(lo), float(hi), mask, 0)


def _noise_range(name: str, value):
    """(low, high) float32 of one servo-noise level: a standard deviation ``s`` or a ``(low, high)`` range"""
    if isinstance(value, (int, float, np.integer, np.floating)):
        lo = hi = value
    else:
        try:
            lo, hi = value
        except (TypeError, ValueError):
            raise UpkieException(f"servo_noise: {name}: expected a standard deviation or a (low, high) pair, got "
                                 f"{value!r}") from None
    try:
        lo, hi = np.float32(lo), np.float32(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"servo_noise: {name}: expected numbers, got ({lo!r}, {hi!r})") from None
    cap = np.float32(_abi.SERVO_NOISE_MAX[name.split(".")[0]])
    if not (np.isfinite(lo) and np.isfinite(hi)) or lo < 0 or hi > cap:
        raise UpkieException(f"servo_noise: {name}: expected finite levels within [0, {cap}], got ({lo}, {hi})")
    if lo > hi:
        raise UpkieException(f"servo_noise: {name}: expected low <= high, got ({lo}, {hi})")
    return lo, hi


def servo_noise_spec(noise, spine_mode: bool = False, joint_limits: Union[bool, int] = True,
                     body_contacts: Union[bool, int] = False, observation_delay: bool = False,
                     servo_dropout: bool = False) -> Optional[_abi.UpkieServoNoise]:
    """``UpkieServoNoise`` (``UpkieSim.set_servo_noise``) from a dict with keys ``position`` (radians) and
    ``velocity`` (rad/s), each a standard deviation ``s`` for every joint, a ``(low, high)`` range from which every
    reset draws each joint's, or a dict ``{joint: s or (low, high)}`` (``JOINT_NAMES``; the joints it leaves out have
    no noise). A quantity left out has no noise. Raises ``UpkieException`` on an unknown key or joint, a level that is
    not a finite number, a negative low, ``low > high``, a position level above 0.1 rad or a velocity level above
    5 rad/s (a sensor noise, not a broken encoder), ``spine_mode`` (whose spine reports its own servos), no joint limits,
    ``body_contacts`` (the noise runs in the kernels of the observation delay), and an observation delay together with
    servo dropouts."""
    if noise is None:
        return None
    if not isinstance(noise, dict):
        raise UpkieException(f"servo_noise: expected a dict with keys 'position' and 'velocity', got {noise!r}")
    unknown = [k for k in noise if k not in ("position", "velocity")]
    if unknown:
        raise UpkieException(f"servo_noise: unknown key(s) {unknown}, expected 'position' and 'velocity'")
    spec = _abi.UpkieServoNoise()
    for name in ("position", "velocity"):
        value = noise.get(name)
        lo = np.zeros(_abi.NJ, dtype=np.float32)
        hi = np.zeros(_abi.NJ, dtype=np.float32)
        if isinstance(value, dict):
            bad = [j for j in value if j not in _abi.JOINT_NAMES]
            if bad:
                raise UpkieException(f"servo_noise: {name}: unknown joint(s) {bad}, expected names of "
                                     f"{_abi.JOINT_NAMES}")
            for j, v in value.items():
                k = _abi.JOINT_NAMES.index(j)
                lo[k], hi[k] = _noise_range(f"{name}.{j}", v)
        elif value is not None:
            lo[:], hi[:] = _noise_range(name, value)
        getattr(spec, f"{name}_low")[:] = [float(x) for x in lo]
        getattr(spec, f"{name}_high")[:] = [float(x) for x in hi]
    if spine_mode:
        raise UpkieException("servo_noise: spine_mode reports the spine's own servos; the noise is not available there")
    if not joint_limits:
        raise UpkieException("servo_noise: needs joint_limits (the noise runs in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("servo_noise: body_contacts has no servo-noise kernels")
    if observation_delay and servo_dropout:
        raise UpkieException("servo_noise: not with both an observation delay and servo dropouts (a delayed snapshot "
                             "does not record which of its replies were held)")
    return spec


# The velocity limits every Upkie's servos are configured with (the reference's tools/configure_servos,
# configure_velocity_limits: servo.max_velocity 2 rev/s on the hips and knees, 8 rev/s on the wheels), and the moteus
# default derate band of 2 rev/s (an assumption, see _abi.MOTEUS_MAX_VELOCITY_DERATE), in rad/s: a ``velocity_derate``
# of ``B200VectorEnv``. 12.57 rad/s on the legs, 50.27 rad/s on the wheels (2.51 m/s of ground velocity).
UPKIE_VELOCITY_DERATE = {
    "max_velocity": {name: (8.0 if "wheel" in name else 2.0) * _abi.RAD_PER_REV for name in _abi.JOINT_NAMES},
    "derate": _abi.MOTEUS_MAX_VELOCITY_DERATE,
}


def _positive_range(name: str, value):
    """(low, high) float32 of one velocity limit: a limit ``v`` or a ``(low, high)`` range, 0 < low <= high"""
    if isinstance(value, (int, float, np.integer, np.floating)):
        lo = hi = value
    else:
        try:
            lo, hi = value
        except (TypeError, ValueError):
            raise UpkieException(f"velocity_derate: {name}: expected a limit or a (low, high) pair, got {value!r}") \
                from None
    try:
        lo, hi = np.float32(lo), np.float32(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"velocity_derate: {name}: expected numbers, got ({lo!r}, {hi!r})") from None
    if not (np.isfinite(lo) and np.isfinite(hi)) or not lo > 0:
        raise UpkieException(f"velocity_derate: {name}: expected finite limits > 0 rad/s, got ({lo}, {hi})")
    if lo > hi:
        raise UpkieException(f"velocity_derate: {name}: expected low <= high, got ({lo}, {hi})")
    return lo, hi


def velocity_derate_spec(velocity_derate, joints=None, spine_mode: bool = False,
                         joint_limits: Union[bool, int] = True,
                         body_contacts: Union[bool, int] = False) -> Optional[_abi.UpkieVelocityDerate]:
    """``UpkieVelocityDerate`` (``UpkieSim.set_velocity_derate``) from a dict with keys ``max_velocity`` and
    ``derate`` (optional, default ``_abi.MOTEUS_MAX_VELOCITY_DERATE``), in rad/s (rev/s times ``2 pi``; see
    ``UPKIE_VELOCITY_DERATE``). ``max_velocity`` is a limit ``v``, a ``(low, high)`` range from which every reset draws
    each joint's limit, or a dict ``{joint: v or (low, high)}``; ``derate`` a band or a dict ``{joint: band}``.
    ``joints`` (names, ``JOINT_NAMES``) are the joints that have a limit; None: the joints of a per-joint
    ``max_velocity``, or all six. Raises ``UpkieException`` on an unknown key or joint, a limit or band that is not a
    finite number > 0, ``low > high``, a joint without a limit, an empty joint list, ``spine_mode`` (whose spine applies
    its own torque law), no joint limits and ``body_contacts`` (the limits run in the kernels of the observation
    delay)."""
    if velocity_derate is None:
        return None
    if not isinstance(velocity_derate, dict) or "max_velocity" not in velocity_derate:
        raise UpkieException(f"velocity_derate: expected a dict with keys 'max_velocity' and 'derate', got "
                             f"{velocity_derate!r}")
    unknown = [k for k in velocity_derate if k not in ("max_velocity", "derate")]
    if unknown:
        raise UpkieException(f"velocity_derate: unknown key(s) {unknown}, expected 'max_velocity' and 'derate'")
    mv = velocity_derate["max_velocity"]
    per_joint = isinstance(mv, dict)
    names = (list(mv) if per_joint else list(_abi.JOINT_NAMES)) if joints is None else list(joints)
    bad = [j for j in names + (list(mv) if per_joint else []) if j not in _abi.JOINT_NAMES]
    if bad:
        raise UpkieException(f"velocity_derate: unknown joint(s) {bad}, expected names of {_abi.JOINT_NAMES}")
    if not names:
        raise UpkieException("velocity_derate_joints: at least one joint")
    spec = _abi.UpkieVelocityDerate()
    lo = np.ones(_abi.NJ, dtype=np.float32)
    hi = np.ones(_abi.NJ, dtype=np.float32)
    band = np.ones(_abi.NJ, dtype=np.float32)
    d = velocity_derate.get("derate", _abi.MOTEUS_MAX_VELOCITY_DERATE)
    if isinstance(d, dict):
        bad = [j for j in d if j not in _abi.JOINT_NAMES]
        if bad:
            raise UpkieException(f"velocity_derate: derate: unknown joint(s) {bad}, expected names of "
                                 f"{_abi.JOINT_NAMES}")
    for j in names:
        k = _abi.JOINT_NAMES.index(j)
        if per_joint and j not in mv:
            raise UpkieException(f"velocity_derate: {j} has no max_velocity")
        lo[k], hi[k] = _positive_range(f"max_velocity.{j}" if per_joint else "max_velocity", mv[j] if per_joint else mv)
        dj = d.get(j, _abi.MOTEUS_MAX_VELOCITY_DERATE) if isinstance(d, dict) else d
        try:
            band[k] = np.float32(dj)
        except (TypeError, ValueError):
            raise UpkieException(f"velocity_derate: derate: expected a number, got {dj!r}") from None
        if not (np.isfinite(band[k]) and band[k] > 0):
            raise UpkieException(f"velocity_derate: derate: expected a finite band > 0 rad/s, got {band[k]}")
    if spine_mode:
        raise UpkieException("velocity_derate: spine_mode applies the spine's own torque law; the limits are not "
                             "available there")
    if not joint_limits:
        raise UpkieException("velocity_derate: needs joint_limits (the limits run in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("velocity_derate: body_contacts has no velocity-limit kernels")
    spec.max_velocity_low[:] = [float(x) for x in lo]
    spec.max_velocity_high[:] = [float(x) for x in hi]
    spec.derate[:] = [float(x) for x in band]
    spec.joint_mask = sum(1 << _abi.JOINT_NAMES.index(j) for j in set(names))
    return spec


def _set_velocity_derate(sim, spec: Optional[_abi.UpkieVelocityDerate]) -> None:
    if spec is None:
        sim.set_velocity_derate(None)
    else:
        sim.set_velocity_derate(list(zip(spec.max_velocity_low, spec.max_velocity_high)), list(spec.derate),
                                [n for j, n in enumerate(_abi.JOINT_NAMES) if (spec.joint_mask >> j) & 1])


def _scale_range(name: str, value):
    """(low, high) float32 of one torque scale: a scale ``s`` or a ``(low, high)`` range, 0 < low <= high <= 2"""
    if isinstance(value, (int, float, np.integer, np.floating)):
        lo = hi = value
    else:
        try:
            lo, hi = value
        except (TypeError, ValueError):
            raise UpkieException(f"torque_scale: {name}: expected a scale or a (low, high) pair, got {value!r}") \
                from None
    try:
        lo, hi = np.float32(lo), np.float32(hi)
    except (TypeError, ValueError):
        raise UpkieException(f"torque_scale: {name}: expected numbers, got ({lo!r}, {hi!r})") from None
    if not (np.isfinite(lo) and np.isfinite(hi)) or not lo > 0 or not hi <= _abi.TORQUE_SCALE_MAX:
        raise UpkieException(f"torque_scale: {name}: expected finite scales in (0, {_abi.TORQUE_SCALE_MAX:g}], got "
                             f"({lo}, {hi})")
    if lo > hi:
        raise UpkieException(f"torque_scale: {name}: expected low <= high, got ({lo}, {hi})")
    return lo, hi


def torque_scale_spec(torque_scale, joints=None, spine_mode: bool = False, joint_limits: Union[bool, int] = True,
                      body_contacts: Union[bool, int] = False) -> Optional[_abi.UpkieTorqueScale]:
    """``UpkieTorqueScale`` (``UpkieSim.set_torque_scale``) from a scale ``s``, a ``(low, high)`` range from which every
    reset draws each joint's scale, or a dict ``{joint: s or (low, high)}`` (dimensionless; ``(0.9, 1.1)`` is a usual
    "motor strength" range in legged-robot RL, not a measured figure of the Upkie's servos). ``joints`` (names,
    ``JOINT_NAMES``) are the joints whose delivered torque is scaled; None: the joints of a dict, or all six. Raises
    ``UpkieException`` on an unknown joint, a scale that is not a finite number in ``(0, 2]``, ``low > high``, a joint
    without a scale, an empty joint list, ``spine_mode`` (whose spine applies its own torque law), no joint limits and
    ``body_contacts`` (the scales run in the kernels of the observation delay)."""
    if torque_scale is None:
        return None
    per_joint = isinstance(torque_scale, dict)
    names = (list(torque_scale) if per_joint else list(_abi.JOINT_NAMES)) if joints is None else list(joints)
    bad = [j for j in names + (list(torque_scale) if per_joint else []) if j not in _abi.JOINT_NAMES]
    if bad:
        raise UpkieException(f"torque_scale: unknown joint(s) {bad}, expected names of {_abi.JOINT_NAMES}")
    if not names:
        raise UpkieException("torque_scale_joints: at least one joint")
    lo = np.ones(_abi.NJ, dtype=np.float32)
    hi = np.ones(_abi.NJ, dtype=np.float32)
    for j in names:
        k = _abi.JOINT_NAMES.index(j)
        if per_joint and j not in torque_scale:
            raise UpkieException(f"torque_scale: {j} has no scale")
        lo[k], hi[k] = _scale_range(j if per_joint else "scale", torque_scale[j] if per_joint else torque_scale)
    if spine_mode:
        raise UpkieException("torque_scale: spine_mode applies the spine's own torque law; the scales are not "
                             "available there")
    if not joint_limits:
        raise UpkieException("torque_scale: needs joint_limits (the scales run in the kernels with joint-limit rows)")
    if body_contacts:
        raise UpkieException("torque_scale: body_contacts has no torque-scale kernels")
    spec = _abi.UpkieTorqueScale()
    spec.scale_low[:] = [float(x) for x in lo]
    spec.scale_high[:] = [float(x) for x in hi]
    spec.joint_mask = sum(1 << _abi.JOINT_NAMES.index(j) for j in set(names))
    return spec


def _set_torque_scale(sim, spec: Optional[_abi.UpkieTorqueScale]) -> None:
    if spec is None:
        sim.set_torque_scale(None)
    else:
        sim.set_torque_scale(list(zip(spec.scale_low, spec.scale_high)),
                             [n for j, n in enumerate(_abi.JOINT_NAMES) if (spec.joint_mask >> j) & 1])


def _set_servo_noise(sim, spec: Optional[_abi.UpkieServoNoise]) -> None:
    if spec is None:
        sim.set_servo_noise(None)
    else:
        sim.set_servo_noise((list(spec.position_low), list(spec.position_high)),
                            (list(spec.velocity_low), list(spec.velocity_high)))


def _set_encoder_offset(sim, spec: Optional[_abi.UpkieEncoderOffset]) -> None:
    if spec is None:
        sim.set_encoder_offset(None)
    else:
        sim.set_encoder_offset(spec.low, spec.high, [n for j, n in enumerate(_abi.JOINT_NAMES)
                                                     if (spec.joint_mask >> j) & 1])


def _set_imu_misalignment(sim, spec: Optional[_abi.UpkieImuMisalignment]) -> None:
    if spec is None:
        sim.set_imu_misalignment(None)
    else:
        sim.set_imu_misalignment((spec.roll_low, spec.roll_high), (spec.pitch_low, spec.pitch_high),
                                 (spec.yaw_low, spec.yaw_high))


class B200VectorEnv(VectorEnv):
    """N Upkie environments stepped by one kernel launch per ``step()``.

    ``max_episode_steps=T`` (0 = none) is Gymnasium's ``TimeLimit`` per env, kept by the step kernel: ``truncated[i]``
    is 1 once env ``i`` has run T steps since its last reset, independently of ``terminated``. The auto-reset fires on
    ``terminated | truncated``; with ``autoreset_mode="disabled"`` an env stays truncated until it is reset.

    With ``autoreset_mode="same_step"``, a step in which some env reset adds ``info["final_obs"]``, the observation
    each resetting env reached before its reset, and ``info["_final_obs"]``, the bool mask of those envs
    (``terminated | truncated``). Unlike ``SyncVectorEnv``'s per-env object array, ``final_obs`` is dense batched
    storage with the observation's structure (servo dictionary of arrays, array, or CUDA tensor from
    ``step_tensors``): rows outside the mask hold stale values. ``base_velocity`` envs (``UpkieBaseVelocity``) take all three
    modes: their ``final_obs`` is the ``[x, y, yaw]`` an env reached, and a reset (fused or through ``reset_mask``)
    also zeroes that env's ``x, y`` and drops its MPC balancer's state. ``copy=True`` copies it as it copies the
    observation. The same step adds the terminal step's info in Gymnasium's layout: ``info["final_info"] =
    {"spine_observation": ..., "_spine_observation": mask}`` and ``info["_final_info"] = mask``. Its
    ``spine_observation`` is a lazy ``FinalSpineObservations``, the same kind of object as ``info["spine_observation"]``
    (``[i]`` the reference's dictionary, ``.array``, ``.tensor``): for each env that reset, the spine observation the
    step led to before the reset, which reward and termination wrappers read. Read it before the next ``step()``.

    Domain randomisation of the actuators: ``torque_control_kp`` / ``torque_control_kd`` take a float or an ``[N]``
    array, ``joint_properties`` a ``{joint: JointProperties}`` dict whose fields are floats or ``[N]`` arrays, or a
    sequence of N such dicts (one per env, as N reference envs would be built). Per-env values go to the handle's
    parameter table (``UpkieSim.set_env_params``, which also takes per-env IMU uncertainty); all-scalar arguments
    build none. ``set_joint_properties`` changes them between episodes.

    ``reset_randomization`` (a dict, see ``reset_randomization_spec``) redraws the given actuator, IMU, inertia and
    floor-friction parameters of an env on the device at every reset of that env, fused auto-resets included: the
    per-episode randomisation a reset wrapper around each env of a ``SyncVectorEnv`` would do. The draws are keyed on
    the seed of ``reset(seed=s)``, which also restarts the draw counters of the envs it resets, so a seeded run repeats.
    ``set_reset_randomization`` changes or (``None``) stops it.

    ``push_randomization`` (a dict, see ``push_randomization_spec``) pushes every env on one link at random times by
    random world-frame forces, scheduled and applied inside the step kernel from each env's own resets: the loop around
    ``set_external_forces`` of the reference's ``apply_external_forces.py``, without a host round trip per step. The
    pushes add to the forces of ``set_external_forces``. They are keyed on the seed of ``reset(seed=s)``, which also
    restarts the schedules of the envs it resets. ``set_push_randomization`` changes or (``None``) stops them.

    ``action_delay`` (seconds, a float or a ``(low, high)`` range, see ``action_delay_spec``) delays each env's servo
    command by a number of substeps drawn at every reset of that env, up to one tick (or ``max_delay_ticks``): the substeps before it run the
    command of the previous tick, and the first ones of an episode run with the servos stopped. The draws are keyed on
    the seed of ``reset(seed=s)``, which also restarts the draw counters of the envs it resets.
    ``set_action_delay`` changes or (``None``) stops it from each env's next reset.

    ``observation_delay`` (seconds, a float or a ``(low, high)`` range, see ``observation_delay_spec``) makes each env
    observe its robot a number of substeps before the end of the tick, drawn at every reset of that env, up to one
    tick (or ``max_delay_ticks``): the observation (and ``base_velocity``'s, through its gyropod rows) describes the robot at that instant,
    while terminations and resets judge the true state; the observation of a reset is undelayed. The draws are keyed on
    the seed of ``reset(seed=s)``, which also restarts the draw counters of the envs it resets.
    ``set_observation_delay`` changes or (``None``) stops it from each env's next reset.

    ``max_delay_ticks`` (1 to ``MAX_DELAY_TICKS``, default 1) is the history both delays keep, in ticks: with it each
    delay may reach ``max_delay_ticks`` ticks instead of one (at ``frequency=1000.0`` a tick is one substep, so the
    default caps each delay at 1 ms). A delay of ``q`` whole ticks and ``r`` substeps runs the command of ``q`` ticks
    earlier from substep ``r``, and reports what a delay of ``r`` substeps reported ``q`` ticks earlier (the state of
    the last reset for the ticks before it). ``set_action_delay`` and ``set_observation_delay`` take the same depth.
    Under an observation delay of a tick or more, the first ticks of an episode report its post-reset state, whose
    measured torques a reset leaves as the previous episode ended them (its zero-torque substep does not write them, as
    for the undelayed reset observation): ``reset(seed=s)`` of a used env then reproduces the physics and every later
    observation, but not those first torque readings; a fresh env reproduces them too.

    ``history`` (key paths of the spine observation, see ``history_spec``) with ``history_size=K`` records those keys
    after every physics substep, as a ``HistoryObserver`` in the spine's pipeline records them every 1 kHz cycle:
    ``info["spine_observation"].history`` is the ``[N, K, C]`` CUDA tensor and ``info["spine_observation"][i]["history"]``
    the reference's ``observation["history"]`` subtree, newest first. Entry 0 is the instant the observation reports
    (under an observation delay too); the IMU accelerations differentiate over one substep and the torques carry no
    measurement noise. Each reset of an env fills its history with the post-reset values (the reference keeps it across
    a spine reset). The terminal step of a same-step reset keeps no history. ``set_history`` changes or (``None``)
    stops it. The history changes no other output.

    ``servo_dropout`` (a probability, or a ``(low, high)`` range, see ``servo_dropout_spec``) loses each reply of the
    servos ``servo_dropout_joints`` (names, default all six) in each 1 kHz spine cycle with a probability drawn at every
    reset of the env, as the spine skips a reply that did not arrive intact (``observe_servos.cpp``): a servo whose reply
    is lost reports the position, velocity and torque of its last received one, in the observation of every env type
    (the gyropod and pendulum wheel odometry too), the spine observation and the history. The physics, terminations
    and ``get_state`` see the true state. The draws are keyed on the seed of ``reset(seed=s)``, which also restarts the
    draw counters of the envs it resets. ``set_servo_dropout`` changes or (``None``) stops it.

    ``imu_misalignment`` (a dict of ``roll`` / ``pitch`` / ``yaw`` angles or ``(low, high)`` ranges in radians, see
    ``imu_misalignment_spec``) mounts each env's IMU off its nominal pose by a rotation drawn at every reset of the env,
    while the observers still assume the nominal ``rotation_base_to_imu`` (``BaseOrientation.h``): the base pitch, its
    rate and rotation, the IMU orientation, rates and accelerations that every env type observes (the gyropod and
    pendulum pitch and pitch rate, the spine observation, the history) are those the tilted IMU reports. The physics,
    terminations and ``get_state`` see the true state. The draws are keyed on the seed of ``reset(seed=s)``, which also
    restarts the draw counters of the envs it resets. ``set_imu_misalignment`` changes or (``None``) stops it.

    ``encoder_offset`` (a bound ``b`` for ``(-b, b)``, or a ``(low, high)`` range in radians, see
    ``encoder_offset_spec``) zeroes the servos ``encoder_offset_joints`` (names, default the hips and knees) off by an
    offset drawn per joint at every reset of the env, as a leg rezeroed by hand would be (``pi3hat_spine.cpp``). The
    servo frame is the joint frame shifted by the offset: every position an env type observes (servo rows, the gyropod
    and pendulum wheel odometry, the spine observation, the history) is ``q + delta``, every position target lands at
    ``target - delta``, and the gyropod, pendulum and base-velocity legs hold their servo zero, the physical angle
    ``-delta``. The physics, terminations and ``get_state``'s q see the true joints. The draws are keyed on the seed of
    ``reset(seed=s)``, which also restarts the draw counters of the envs it resets. ``set_encoder_offset`` changes or
    (``None``) stops it.

    ``servo_noise`` (a dict ``{"position": ..., "velocity": ...}``, each a standard deviation, a ``(low, high)`` range
    or ``{joint: s or (low, high)}``, see ``servo_noise_spec``) adds white noise to every servo position (radians) and
    velocity (rad/s) reply, at levels drawn per joint at every reset of the env, as the moteus encoder estimates reach
    the spine (``observe_servos.cpp``). Every position and velocity an env type observes (servo rows, the gyropod and
    pendulum wheel odometry, the spine observation, the history) carries the noise of the spine cycle it reports; the
    physics, the torques, terminations and ``get_state`` see the true replies. The draws are keyed on the seed of
    ``reset(seed=s)``, which also restarts the draw counters of the envs it resets. ``set_servo_noise`` changes or
    (``None``) stops it.

    ``velocity_derate`` (a dict ``{"max_velocity": ..., "derate": ...}`` in rad/s, see ``velocity_derate_spec``;
    ``UPKIE_VELOCITY_DERATE`` holds the robot's configured 2 rev/s legs and 8 rev/s wheels, a rev/s being ``2 pi``
    rad/s) limits the servos ``velocity_derate_joints`` (names, default those of ``max_velocity``) as the moteus
    ``servo.max_velocity`` does: past a limit drawn per joint at every reset of the env, the torque that drives a joint
    faster falls linearly to zero over the derate band, while a braking torque passes. The torque every env type
    observes is the derated one. The draws are keyed on the seed of ``reset(seed=s)``, which also restarts the draw
    counters of the envs it resets. ``set_velocity_derate`` changes or (``None``) stops it.

    ``torque_scale`` (a scale, a ``(low, high)`` range or ``{joint: s or (low, high)}``, see ``torque_scale_spec``)
    makes the servos ``torque_scale_joints`` (names, default those of a dict, or all six) deliver a scale of the torque
    they command, drawn per joint at every reset of the env, as a servo whose torque constant is off: the physics
    integrates the scaled torque, while the torque every env type observes stays the commanded one. ``(0.9, 1.1)`` is a
    usual range in legged-robot RL, not a measured tolerance of the Upkie's servos. The draws are keyed on the seed of
    ``reset(seed=s)``, which also restarts the draw counters of the envs it resets. ``set_torque_scale`` changes or
    (``None``) stops it.

    ``attitude_filter`` (a dict ``{"kp": ..., "ki": ..., "roll": ..., "pitch": ...}``, see ``attitude_filter_spec``)
    makes every env report the orientation an attitude filter estimates from its simulated IMU, as the robot's spine
    reads the pi3hat's filter: the IMU orientation, the base pitch and rotation, and the gyropod and pendulum pitch
    carry the filter's convergence, its tilt error under acceleration and its drift from gyro bias, while the rates,
    accelerations, physics and terminations do not. Every reset of an env draws its gains and an initial estimate error;
    the draws are keyed on the seed of ``reset(seed=s)``, which also restarts the draw counters of the envs it resets.
    ``set_attitude_filter`` changes or (``None``) stops it.
    """

    metadata: Dict[str, Any] = {"autoreset_mode": "disabled"}

    def __init__(
        self,
        num_envs: int,
        env_type: str = "servos",
        frequency: float = 200.0,
        init_state: Optional[RobotState] = None,
        model: Optional[Model] = None,
        device: int = 0,
        autoreset_mode: str = "disabled",
        max_gain_scale: float = 5.0,
        fall_pitch: float = 1.0,
        leg_gain_scale: float = 1.0,
        max_ground_velocity: float = 3.0,
        max_yaw_velocity: float = 1.0,
        nb_substeps: Optional[int] = None,
        torque_control_kp: Union[float, np.ndarray] = 20.0,
        torque_control_kd: Union[float, np.ndarray] = 1.0,
        joint_properties: Optional[Union[dict, Sequence[dict]]] = None,
        inertia_variation: float = 0.0,
        env_offset: int = 0,
        config: Optional[_abi.UpkieSimConfig] = None,
        leg_length: float = 0.58,
        max_ground_accel: float = 10.0,
        noise_seed: int = 0,
        joint_limits: Union[bool, int] = True,
        copy: bool = True,
        spine_mode: bool = False,
        body_contacts: bool = False,
        max_episode_steps: int = 0,
        reset_randomization: Optional[dict] = None,
        push_randomization: Optional[dict] = None,
        action_delay: Optional[Union[float, Tuple[float, float]]] = None,
        observation_delay: Optional[Union[float, Tuple[float, float]]] = None,
        max_delay_ticks: int = 1,
        history=None,
        history_size: int = 1,
        servo_dropout: Optional[Union[float, Tuple[float, float]]] = None,
        servo_dropout_joints: Optional[Sequence[str]] = None,
        imu_misalignment: Optional[Dict[str, Union[float, Tuple[float, float]]]] = None,
        encoder_offset: Optional[Union[float, Tuple[float, float]]] = None,
        encoder_offset_joints: Optional[Sequence[str]] = None,
        servo_noise: Optional[Dict[str, Any]] = None,
        velocity_derate: Optional[Dict[str, Any]] = None,
        velocity_derate_joints: Optional[Sequence[str]] = None,
        attitude_filter: Optional[Dict[str, Any]] = None,
        torque_scale: Optional[Union[float, Tuple[float, float], Dict[str, Any]]] = None,
        torque_scale_joints: Optional[Sequence[str]] = None,
    ):
        max_episode_steps = _check_max_episode_steps(max_episode_steps)
        rr_spec = reset_randomization_spec(reset_randomization)  # validated before any device is touched
        push_spec = push_randomization_spec(push_randomization, model if model is not None else default_model(),
                                            1.0 / frequency)
        if env_type not in ENV_TYPES:
            raise UpkieException(f"env_type must be one of {ENV_TYPES}")
        if autoreset_mode not in _AUTORESET:
            raise UpkieException(f"autoreset_mode must be one of {tuple(_AUTORESET)}")
        self.env_type = env_type
        # host path: ``step()`` results live in the handle's pinned output buffers, which the next ``step()``
        # overwrites. copy=True (default, as gymnasium.vector.SyncVectorEnv(copy=True)) hands out copies, so that
        # ``buf.append(obs)`` or ``prev_obs`` comparisons do not alias; copy=False returns views of the pinned buffers
        # (zero-copy fast path, valid until the next step; what bench.py's e2e figure uses and says so)
        self.copy = bool(copy)
        self.num_envs = int(num_envs)
        self.model = model if model is not None else default_model()
        self.init_state = init_state if init_state is not None else RobotState(
            position_base_in_world=np.array([0.0, 0.0, 0.6])
        )
        self.frequency = frequency
        self.dt = 1.0 / frequency
        self.env_offset = int(env_offset)
        self.autoreset_mode = autoreset_mode
        self.metadata = dict(self.metadata, autoreset_mode=autoreset_mode)
        per_env = needs_env_params(torque_control_kp, torque_control_kd, joint_properties)
        if config is None:
            # per-env arguments go to the parameter table below; the config keeps the scalar ones
            config = make_config(
                frequency, nb_substeps,
                20.0 if _per_env(torque_control_kp) else torque_control_kp,
                1.0 if _per_env(torque_control_kd) else torque_control_kd,
                None if per_env else joint_properties, max_gain_scale,
                fall_pitch, leg_gain_scale, max_ground_velocity, max_yaw_velocity, self.init_state, noise_seed,
                joint_limits, spine_mode, body_contacts, max_episode_steps,
            )
        elif max_episode_steps:
            # an explicit limit overrides the one of the given configuration (a copy: the caller's struct is untouched)
            config = _abi.UpkieSimConfig.from_buffer_copy(config)
            config.max_episode_steps = max_episode_steps
        self.config = config
        self.max_delay_ticks = _check_max_delay_ticks(max_delay_ticks)
        delay_spec = action_delay_spec(action_delay, 1.0 / frequency, config.nb_substeps, bool(config.spine_mode),
                                       config.joint_limits, self.max_delay_ticks)  # validated before any device is touched
        sense_spec = observation_delay_spec(observation_delay, 1.0 / frequency, config.nb_substeps,
                                            bool(config.spine_mode), config.joint_limits, config.body_contacts,
                                            self.max_delay_ticks)  # validated before any device is touched
        hist_spec = history_spec(history, history_size, bool(config.spine_mode), config.joint_limits,
                                 bool(config.body_contacts))  # validated before any device is touched
        drop_spec = servo_dropout_spec(servo_dropout, servo_dropout_joints, bool(config.spine_mode),
                                       config.joint_limits, config.body_contacts)  # validated before any device
        tilt_spec = imu_misalignment_spec(imu_misalignment, bool(config.spine_mode), config.joint_limits,
                                          config.body_contacts)  # validated before any device is touched
        enc_spec = encoder_offset_spec(encoder_offset, encoder_offset_joints, bool(config.spine_mode),
                                       config.joint_limits, config.body_contacts)  # validated before any device
        noise_spec = servo_noise_spec(servo_noise, bool(config.spine_mode), config.joint_limits, config.body_contacts,
                                      sense_spec is not None, drop_spec is not None)  # validated before any device
        att_spec = attitude_filter_spec(attitude_filter, bool(config.spine_mode), config.joint_limits,
                                        config.body_contacts, 1.0 / frequency, config.nb_substeps,
                                        self.max_delay_ticks if sense_spec is not None else 1)  # before any device
        vlim_spec = velocity_derate_spec(velocity_derate, velocity_derate_joints, bool(config.spine_mode),
                                         config.joint_limits, config.body_contacts)  # validated before any device
        tsc_spec = torque_scale_spec(torque_scale, torque_scale_joints, bool(config.spine_mode), config.joint_limits,
                                     config.body_contacts)  # validated before any device is touched
        # validated before any device is touched
        env_params = env_params_table(self.num_envs, _abi.config_env_params(config), torque_control_kp,
                                      torque_control_kd, joint_properties) if per_env else None
        if self.config.spine_mode and env_type != "servos":
            raise UpkieException("spine_mode is available for env_type='servos' (the wrappers of a spine read observer "
                                 "outputs: feed info['spine_observation'] to upkie_b200.observers.ObserverPipeline)")
        (
            servo_act, servo_obs, self._neutral_action, self._max_action, self._min_action,
        ) = make_servo_spaces(self.model, max_gain_scale)
        if env_type == "servos":
            self.single_action_space, self.single_observation_space = servo_act, servo_obs
        elif env_type == "gyropod":
            self.single_action_space, self.single_observation_space = make_gyropod_spaces(
                max_ground_velocity, max_yaw_velocity
            )
        elif env_type == "base_velocity":
            self.single_action_space, self.single_observation_space = make_base_velocity_spaces(
                max_ground_velocity, max_yaw_velocity
            )
        else:
            self.single_action_space, self.single_observation_space = make_pendulum_spaces(max_ground_velocity)
        self.action_space = batch_space(self.single_action_space, self.num_envs)
        self.observation_space = batch_space(self.single_observation_space, self.num_envs)

        self.sim = UpkieSim(self.num_envs, model=self.model, config=self.config, device=device)
        if env_params is not None:
            self.sim.set_env_params(torch.from_numpy(env_params).to(self.sim.device))
        self._seed = 0
        self.mpc_balancer = None
        if env_type == "base_velocity":
            # UpkieBaseVelocity embeds an MPCBalancer (upkie_base_velocity.py:117-126)
            from .mpc import BatchedMPCBalancer

            self.mpc_balancer = BatchedMPCBalancer(
                self.num_envs, fall_pitch=fall_pitch, leg_length=leg_length, max_ground_accel=max_ground_accel,
                max_ground_velocity=max_ground_velocity, device=device,
            )
            self._xy = torch.zeros((self.num_envs, 2), dtype=torch.float32, device=self.sim.device)
            self._spine = None
            self._bv_obs = None  # the observation the last step / reset returned (device), None = zeros
        self.sim.set_autoreset(_AUTORESET[autoreset_mode], self._seed, self.env_offset)
        self.inertia_variation = inertia_variation
        if abs(inertia_variation) > 1e-10:
            self.randomize_inertias(inertia_variation)
        if rr_spec is not None:
            self.sim.set_reset_randomization(rr_spec)
        if push_spec is not None:
            self.sim.set_push_randomization(push_spec)
        if delay_spec is not None:
            # before the first reset, which draws every env's delay
            self.sim.set_action_delay(*delay_spec, max_ticks=self.max_delay_ticks)
        if sense_spec is not None:
            # before the first reset, which draws every env's delay
            self.sim.set_observation_delay(*sense_spec, max_ticks=self.max_delay_ticks)
        self._history_layout = None
        if hist_spec is not None:
            self.sim.set_history(hist_spec[0], hist_spec[1])
            self._history_layout = hist_spec[2]
        if drop_spec is not None:
            # before the first reset, which draws every env's probability
            self.sim.set_servo_dropout(drop_spec.prob_low, drop_spec.prob_high, servo_dropout_joints)
        if tilt_spec is not None:
            _set_imu_misalignment(self.sim, tilt_spec)  # before the first reset, which draws every env's misalignment
        if enc_spec is not None:
            _set_encoder_offset(self.sim, enc_spec)  # before the first reset, which draws every env's offsets
        if noise_spec is not None:
            _set_servo_noise(self.sim, noise_spec)  # before the first reset, which draws every env's levels
        if vlim_spec is not None:
            _set_velocity_derate(self.sim, vlim_spec)  # before the first reset, which draws every env's limits
        if tsc_spec is not None:
            _set_torque_scale(self.sim, tsc_spec)  # before the first reset, which draws every env's scales
        if att_spec is not None:
            _set_attitude_filter(self.sim, att_spec)  # before the first reset, which draws every env's filter

    def set_attitude_filter(self, attitude_filter) -> None:
        """Report every env's orientation from an attitude filter on its IMU, with gains and an initial error drawn per
        env (a dict, see ``attitude_filter_spec``); ``None`` turns the filter off. New ranges take effect at each env's
        next reset; a first filter starts every env from its true orientation with the upper gains."""
        sense = getattr(self.sim, "_observation_delay", None)
        _set_attitude_filter(self.sim, attitude_filter_spec(
            attitude_filter, bool(self.config.spine_mode), self.config.joint_limits, self.config.body_contacts,
            float(self.config.dt), self.config.nb_substeps, self.max_delay_ticks if sense is not None else 1))

    def set_velocity_derate(self, velocity_derate, joints=None) -> None:
        """Limit the servos ``joints`` (names, None: those of ``max_velocity``) past a velocity drawn per env (a dict
        in rad/s, see ``velocity_derate_spec``; ``UPKIE_VELOCITY_DERATE`` for the robot's configuration); ``None``
        turns the limits off. New ranges take effect at each env's next reset; the joints it adds are limited at their
        ``high`` bound until then, and those it drops have no limit from now on."""
        _set_velocity_derate(self.sim, velocity_derate_spec(velocity_derate, joints, bool(self.config.spine_mode),
                                                            self.config.joint_limits, self.config.body_contacts))

    def set_torque_scale(self, torque_scale, joints=None) -> None:
        """Scale the torque the servos ``joints`` (names, None: those of a dict, or all six) deliver by a factor drawn
        per env (see ``torque_scale_spec``); ``None`` turns the scales off. New ranges take effect at each env's next
        reset; the joints it adds hold a scale of 1 until then, and those it drops have none from now on."""
        _set_torque_scale(self.sim, torque_scale_spec(torque_scale, joints, bool(self.config.spine_mode),
                                                      self.config.joint_limits, self.config.body_contacts))

    def set_servo_noise(self, noise) -> None:
        """Add white noise to the servos' position and velocity replies at levels drawn per env (a dict, see
        ``servo_noise_spec``); ``None`` turns the noise off. New ranges take effect at each env's next reset; the
        columns whose range they make zero have no noise from now on."""
        _set_servo_noise(self.sim, servo_noise_spec(noise, bool(self.config.spine_mode), self.config.joint_limits,
                                                    self.config.body_contacts,
                                                    getattr(self.sim, "_observation_delay", None) is not None,
                                                    self.sim.servo_dropout_spec is not None))

    def set_encoder_offset(self, offset, joints=None) -> None:
        """Zero the servos ``joints`` (names, None: the hips and knees) off by an offset drawn from a bound or a
        ``(low, high)`` range in radians (``encoder_offset_spec``); ``None`` turns the offsets off. A new range takes
        effect at each env's next reset; the joints it drops have no offset from now on."""
        _set_encoder_offset(self.sim, encoder_offset_spec(offset, joints, bool(self.config.spine_mode),
                                                          self.config.joint_limits, self.config.body_contacts))

    def set_imu_misalignment(self, misalignment) -> None:
        """Mount each env's IMU off its nominal pose by ``roll`` / ``pitch`` / ``yaw`` angles or ranges (a dict,
        ``imu_misalignment_spec``); ``None`` turns the misalignment off. New ranges take effect at each env's next
        reset."""
        _set_imu_misalignment(self.sim, imu_misalignment_spec(misalignment, bool(self.config.spine_mode),
                                                              self.config.joint_limits, self.config.body_contacts))

    def set_servo_dropout(self, prob, joints=None) -> None:
        """Lose the replies of the servos ``joints`` (names, None: all) with a per-cycle probability ``prob``, a float
        or a ``(low, high)`` range (``servo_dropout_spec``); ``None`` turns the dropouts off. A new range takes effect
        at each env's next reset."""
        spec = servo_dropout_spec(prob, joints, bool(self.config.spine_mode), self.config.joint_limits,
                                  self.config.body_contacts)
        if spec is None:
            self.sim.set_servo_dropout(None)
        else:
            self.sim.set_servo_dropout(spec.prob_low, spec.prob_high, joints)

    def set_history(self, keys, size: int = 1) -> None:
        """Record the spine-observation ``keys`` (``history_spec``) after every substep and report the last ``size``
        in ``info["spine_observation"]``; ``None`` turns the history off. Every env's history restarts from its
        current state."""
        spec = history_spec(keys, size, bool(self.config.spine_mode), self.config.joint_limits,
                            bool(self.config.body_contacts))
        if spec is None:
            self.sim.set_history(None)
            self._history_layout = None
        else:
            self.sim.set_history(spec[0], spec[1])
            self._history_layout = spec[2]

    def _spine_observations(self) -> "SpineObservations":
        return SpineObservations(self.sim, self._history_layout)

    def set_reset_randomization(self, spec: Optional[dict]) -> None:
        """Redraw the parameters ``spec`` names at every later reset of an env (``reset_randomization_spec``);
        ``None`` stops redrawing, the values then in force stay."""
        self.sim.set_reset_randomization(reset_randomization_spec(spec))

    def set_push_randomization(self, spec: Optional[dict]) -> None:
        """Push every env at random times by random forces (``push_randomization_spec``, times in seconds of this
        env's ``dt``); ``None`` stops pushing. Takes effect from the next step; no schedule restarts."""
        self.sim.set_push_randomization(push_randomization_spec(spec, self.model, self.dt))

    def set_action_delay(self, delay) -> None:
        """Delay the servo commands by ``delay`` seconds, a float or a ``(low, high)`` range (``action_delay_spec``);
        ``None`` turns the delay off. A new range takes effect at each env's next reset."""
        spec = action_delay_spec(delay, self.dt, self.config.nb_substeps, bool(self.config.spine_mode),
                                 self.config.joint_limits, self.max_delay_ticks)
        if spec is None:
            self.sim.set_action_delay(None)
        else:
            self.sim.set_action_delay(*spec, max_ticks=self.max_delay_ticks)

    def set_observation_delay(self, delay) -> None:
        """Observe each robot ``delay`` seconds before the end of the tick, a float or a ``(low, high)`` range
        (``observation_delay_spec``); ``None`` turns the delay off. A new range takes effect at each env's next
        reset."""
        spec = observation_delay_spec(delay, self.dt, self.config.nb_substeps, bool(self.config.spine_mode),
                                      self.config.joint_limits, self.config.body_contacts, self.max_delay_ticks)
        if spec is None:
            self.sim.set_observation_delay(None)
        else:
            self.sim.set_observation_delay(*spec, max_ticks=self.max_delay_ticks)

    # ------------------------------------------------------------------
    def get_neutral_action(self) -> dict:
        """``UpkieServos.get_neutral_action`` (``upkie_servos.py:308-314``)."""
        return self._neutral_action.copy()

    def randomize_inertias(self, inertia_variation: float, seed: Optional[int] = None) -> None:
        """``PyBulletBackend.randomize_inertias`` (``pybullet_backend.py:571-601``):
        one epsilon ~ U(-v, v) per non-base body and env."""
        rng = np.random.default_rng(seed)
        eps = rng.uniform(-inertia_variation, inertia_variation, size=(self.num_envs, 6)).astype(np.float32)
        self.sim.set_randomization(inertia_eps=torch.from_numpy(eps).to(self.sim.device))

    def set_joint_properties(self, joint_properties=None, torque_control_kp=None, torque_control_kd=None) -> None:
        """Re-randomise the actuators between episodes, with the constructor's argument forms; what is not given
        (None) keeps its current per-env values. Takes effect from the next step."""
        base = self.sim.get_env_params().cpu().numpy()
        table = env_params_table(self.num_envs, base, torque_control_kp, torque_control_kd, joint_properties)
        self.sim.set_env_params(torch.from_numpy(table).to(self.sim.device))

    def update_init_rand(self, **kwargs) -> None:
        """``UpkieEnv.update_init_rand`` (``upkie_env.py:244-251``)."""
        self.init_state.randomization.update(**kwargs)
        # the fused auto-reset samples on the device: carry the new bounds there too
        self.init_state.apply_to_config(self.config)
        self.sim.set_config(self.config)

    def close(self, **kwargs) -> None:
        self.sim.close()

    # ------------------------------------------------------------------
    def _obs_dim(self) -> int:
        return {"servos": 30, "gyropod": 6, "pendulum": 4, "base_velocity": 6}[self.env_type]

    def _format_obs(self, obs: np.ndarray):
        if self.env_type != "servos":
            return obs
        # the host-path observation lives in one persistent pinned buffer: build the dictionary of
        # views once and hand the same (in-place updated) dictionary back on every step
        cache = getattr(self, "_obs_dict_cache", None)
        if cache is None or cache[0] is not obs:
            cache = (obs, servo_obs_array_to_dict(obs))
            if obs is self.sim._host_buffers()["obs30"]:
                self._obs_dict_cache = cache
        return cache[1]

    def get_contact_points(self, env_index: int = 0, link_name: Optional[str] = None) -> list:
        """``PyBulletBackend.get_contact_points`` (``pybullet_backend.py:660-716``) for one env of the batch."""
        from .model import contact_points_from_state

        row = self.sim.get_state()[int(env_index)].cpu().numpy()
        rec = self.sim.get_body_contacts()[int(env_index)].cpu().numpy()
        return contact_points_from_state(self.model, row, self.config, link_name, rec)

    def set_external_forces(self, external_forces: Optional[dict]) -> None:
        """Batched ``PyBulletBackend.set_external_forces``: ``{link name: ExternalForce}`` whose ``force`` is
        ``[3]`` (all envs) or ``[N, 3]``; ``None`` or ``{}`` clears."""
        if not external_forces:
            self.sim.set_external_forces(None)
            return
        rows, mask = self.model.external_force_rows(external_forces, self.num_envs)
        self.sim.set_external_forces(torch.from_numpy(rows).to(self.sim.device), mask)

    def _servo_obs_dict(self, obs18: np.ndarray, cache: bool = True) -> dict:
        """Batched observation dictionary over the persistent pinned ``[N, 6, 3]`` buffer the kernel writes
        (position, velocity, torque): built once, updated in place by every step. Temperature and voltage
        are the simulator's constants (``pybullet_backend.py:471-472``) and never cross PCIe."""
        cached = getattr(self, "_obs18_cache", None) if cache else None
        if cached is None or cached[0] is not obs18:
            n = self.num_envs
            const = getattr(self, "_obs_constants", None)
            if const is None:
                # pybullet_backend.py:471 (42.0) / BulletInterface.cpp:70 in spine mode (20.0)
                temperature = np.full((n, 1), 20.0 if self.config.spine_mode else 42.0, dtype=np.float32)
                voltage = np.full((n, 1), 18.0, dtype=np.float32)
                temperature.flags.writeable = False
                voltage.flags.writeable = False
                const = self._obs_constants = (temperature, voltage)
            temperature, voltage = const
            d = {
                name: {
                    "position": obs18[:, j, 0:1],
                    "velocity": obs18[:, j, 1:2],
                    "torque": obs18[:, j, 2:3],
                    "temperature": temperature,
                    "voltage": voltage,
                }
                for j, name in enumerate(_abi.JOINT_NAMES)
            }
            cached = (obs18, d)
            if cache:
                self._obs18_cache = cached
        return cached[1]

    def reset(self, *, seed: Optional[Union[int, list]] = None, options: Optional[dict] = None):
        """Reset all envs (or ``options["reset_mask"]``) and return the initial
        observations. Env ``i`` samples its initial state from
        ``np.random.default_rng(seed + i)`` exactly as ``UpkieEnv.reset(seed)``
        does for a single env (``upkie_env.py:180-190``); with ``seed=None``
        the envs draw from the vector env's own generator."""
        n = self.num_envs
        mask = None
        if options and options.get("reset_mask") is not None:
            mask = np.ascontiguousarray(options["reset_mask"], dtype=np.uint8).reshape(n)
        parent = self.np_random
        if seed is None:
            seeds = [None] * n
        elif isinstance(seed, (list, tuple, np.ndarray)):
            seeds = list(seed)
        else:
            seeds = [int(seed) + self.env_offset + i for i in range(n)]
            self._seed = int(seed)
            self.sim.set_autoreset(_AUTORESET[self.autoreset_mode], self._seed, self.env_offset)
            if getattr(self.sim, "_reset_randomization", None) is not None:
                # the reset randomisation is keyed on this seed: the envs reset here draw again from draw 1
                draws = self.sim.get_draws()
                if mask is None:
                    draws.zero_()
                else:
                    draws.masked_fill_(torch.from_numpy(mask).to(draws.device).bool(), 0)
                self.sim.set_draws(draws)
            if getattr(self.sim, "_push_randomization", None) is not None:
                # so is the push schedule: the envs reset here restart from count 0, timer 0 (their reset then
                # makes draw 1)
                count, timer = self.sim.get_push_state()
                if mask is None:
                    count.zero_()
                    timer.zero_()
                else:
                    m = torch.from_numpy(mask).to(count.device).bool()
                    count.masked_fill_(m, 0)
                    timer.masked_fill_(m, 0)
                self.sim.set_push_state(count, timer)
            if getattr(self.sim, "_action_delay", None) is not None:
                # so is the action delay: the envs reset here restart from count 0 (their reset then makes draw 1)
                count, delay, command = self.sim.get_action_delay_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_action_delay_state(count, delay, command)
            if getattr(self.sim, "_observation_delay", None) is not None:
                # so is the observation delay
                count, delay, rows = self.sim.get_observation_delay_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_observation_delay_state(count, delay, rows)
            if self.sim.servo_dropout_spec is not None:
                # so are the servo dropouts
                count, prob, held = self.sim.get_servo_dropout_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_servo_dropout_state(count, prob, held)
            if self.sim.imu_misalignment_spec is not None:
                # so is the IMU misalignment
                count, quat = self.sim.get_imu_misalignment_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_imu_misalignment_state(count, quat)
            if self.sim.encoder_offset_spec is not None:
                # so are the encoder offsets
                count, offset = self.sim.get_encoder_offset_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_encoder_offset_state(count, offset)
            if self.sim.servo_noise_spec is not None:
                # so is the servo noise
                count, sigma = self.sim.get_servo_noise_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_servo_noise_state(count, sigma)
            if self.sim.velocity_derate_spec is not None:
                # so are the velocity limits
                count, vmax = self.sim.get_velocity_derate_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_velocity_derate_state(count, vmax)
            if self.sim.torque_scale_spec is not None:
                # so are the torque scales
                count, scale = self.sim.get_torque_scale_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_torque_scale_state(count, scale)
            if self.sim.attitude_filter_spec is not None:
                # and the attitude filter's draws
                count, gains, quat, bias = self.sim.get_attitude_filter_state()
                if mask is None:
                    count.zero_()
                else:
                    count.masked_fill_(torch.from_numpy(mask).to(count.device).bool(), 0)
                self.sim.set_attitude_filter_state(count, gains, quat, bias)
        rows = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
        for i in range(n):
            if mask is not None and not mask[i]:
                continue
            rng = parent if seeds[i] is None else np.random.default_rng(seeds[i])
            rows[i] = self.init_state.sample_state(rng).to_row()
        dev = self.sim.device
        self.sim.reset(
            mask=torch.from_numpy(mask).to(dev) if mask is not None else None,
            init_state=torch.from_numpy(rows).to(dev),
        )
        info = {"spine_observation": self._spine_observations()}
        if self.env_type == "base_velocity":
            # UpkieBaseVelocity.reset (upkie_base_velocity.py:137-162) of the reset envs: MPC reset, x = y = 0, zero
            # observation; the other envs keep their state and their last observation
            if mask is None:
                self.mpc_balancer.reset()
                self._xy.zero_()
                obs = torch.zeros((n, 3), dtype=torch.float32, device=dev)
            else:
                m = torch.from_numpy(mask).to(dev)
                self.mpc_balancer.reset(m)
                self._xy.masked_fill_(m.bool()[:, None], 0.0)
                obs = torch.zeros((n, 3), dtype=torch.float32, device=dev) if self._bv_obs is None else self._bv_obs.clone()
                obs.masked_fill_(m.bool()[:, None], 0.0)
            self._spine = self.sim.spine_obs()
            self._bv_obs = obs
            return obs.cpu().numpy(), info
        obs = self.sim.reset_obs(self._obs_dim()).cpu().numpy()
        return self._format_obs(obs), info

    def step(self, action):
        """One 5 ms control tick for every env. ``action`` is a batched dict
        (servos), an ndarray / CPU tensor, or a CUDA tensor (then the result
        tensors stay on the device)."""
        if isinstance(action, torch.Tensor) and action.is_cuda:
            return self.step_tensors(action)
        n = self.num_envs
        if self.env_type == "base_velocity":
            a = torch.from_numpy(np.ascontiguousarray(np.asarray(action, dtype=np.float32).reshape(n, 2))).to(self.sim.device)
            obs, rew, term, trunc, info = self.step_tensors(a)
            if "final_obs" in info:  # host copies, as the other env types' host path returns them
                info["final_obs"] = info["final_obs"].cpu().numpy()
                info["_final_obs"] = info["_final_obs"].cpu().numpy()
                info["_final_info"] = info["_final_info"].cpu().numpy()
                fi = info["final_info"]
                fi["_spine_observation"] = fi["_spine_observation"].cpu().numpy()
            return obs.cpu().numpy(), rew.cpu().numpy(), term.cpu().numpy().view(np.bool_), trunc.cpu().numpy().view(np.bool_), info
        if self.env_type == "servos":
            a = (
                servo_action_dict_to_array(action, self._neutral_action, n)
                if isinstance(action, dict)
                else np.ascontiguousarray(np.asarray(action, dtype=np.float32).reshape(n, 6, 6))
            )
            hb = self.sim._host_buffers()
            fin = None
            if self._host_general_step():
                obs18, term, trunc, fin = self.sim.step_host(a, 36, compact=True, final_obs=self._same_step(),
                                                             final_state=self._same_step())
            else:
                obs18, term, trunc = *self.sim.step_servos_host_compact(a), hb["trunc"]
            info = {"spine_observation": self._spine_observations()}
            if self.copy:
                obs18 = obs18.copy()
                self._add_final_obs(info, term, trunc, fin, lambda f: self._servo_obs_dict(f.copy(), cache=False))
                return (self._servo_obs_dict(obs18, cache=False), hb["rew"].copy(), term.view(np.bool_).copy(),
                        trunc.view(np.bool_).copy(), info)
            self._add_final_obs(info, term, trunc, fin, lambda f: self._servo_obs_dict(f, cache=False))
            return self._servo_obs_dict(obs18), hb["rew"], term.view(np.bool_), trunc.view(np.bool_), info
        else:
            d = 2 if self.env_type == "gyropod" else 1
            a = np.ascontiguousarray(np.asarray(action, dtype=np.float32).reshape(n, d))
            fin = None
            if self._host_general_step():
                obs, term, trunc, fin = self.sim.step_host(a, d, final_obs=self._same_step(), final_state=self._same_step())
                rew = self.sim._host_buffers()["rew"]
            else:
                obs, rew, term, trunc = self.sim.step_gyropod_host(a)
        info = {"spine_observation": self._spine_observations()}
        if self.copy:
            self._add_final_obs(info, term, trunc, fin, np.copy)
            return obs.copy(), rew.copy(), term.view(np.bool_).copy(), trunc.view(np.bool_).copy(), info
        # views of the handle's pinned output buffers: valid until the next step()
        self._add_final_obs(info, term, trunc, fin, lambda f: f)
        return self._format_obs(obs), rew, term.view(np.bool_), trunc.view(np.bool_), info

    def _same_step(self) -> bool:
        return self.autoreset_mode == "same_step"

    def _host_general_step(self) -> bool:
        """Host path through ``upkie_b200_step_host`` (``truncated`` from the kernel, final observations) when a time
        limit or the same-step auto-reset needs it; otherwise the calls that leave ``truncated`` on the host."""
        return self.config.max_episode_steps > 0 or self._same_step()

    def _add_final_obs(self, info: dict, term, trunc, fin, fmt) -> None:
        """``info["final_obs"]`` / ``info["_final_obs"]`` and ``info["final_info"]`` / ``info["_final_info"]`` when
        some env reset in this step (same-step mode, whose steps stash the pre-reset states)."""
        if fin is None:
            return
        if isinstance(term, torch.Tensor):
            mask = (term | trunc).bool()
            if not bool(mask.any()):
                return
            copy = torch.clone
        else:
            mask = (term | trunc).view(np.bool_)
            if not mask.any():
                return
            copy = np.copy
        info["final_obs"] = fmt(fin)
        info["_final_obs"] = mask
        # Gymnasium 1.x SyncVectorEnv._add_info layout: a dict of the terminal infos, each key with its `_key` mask
        info["final_info"] = {"spine_observation": FinalSpineObservations(self.sim), "_spine_observation": copy(mask)}
        info["_final_info"] = copy(mask)

    def step_tensors(self, action: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor, dict]:
        """Zero-copy fast path: CUDA tensors in, CUDA tensors out
        (``action[N, 6, 6]`` / ``[N, 2]`` / ``[N, 1]``). In same-step mode ``info["final_obs"]`` is a CUDA tensor of
        the observation's shape and ``info["_final_obs"]`` a CUDA bool tensor."""
        same = self._same_step()
        fin = self._device_final_obs() if same else None
        if self.env_type == "servos":
            obs, rew, term, trunc = self.sim.step_servos(action, final_obs=fin, final_state=same)
        elif self.env_type == "gyropod":
            obs, rew, term, trunc = self.sim.step_gyropod(action, final_obs=fin, final_state=same)
        elif self.env_type == "base_velocity":
            obs, rew, term, trunc = self._base_velocity_step(action, fin)
        else:
            obs, rew, term, trunc = self.sim.step_pendulum(action, final_obs=fin, final_state=same)
        info = {"spine_observation": self._spine_observations()}
        # same-step mode: one host synchronisation per step decides whether some env reset
        self._add_final_obs(info, term, trunc, fin, lambda f: f)
        return obs, rew, term, trunc, info

    def _base_velocity_step(self, action: torch.Tensor, fin: Optional[torch.Tensor]):
        """``UpkieBaseVelocity.step`` (``upkie_base_velocity.py:164-202``) in ``base_velocity_tick``'s order: the MPC
        turns the commanded linear velocity into a ground velocity from the LAST spine observation, the gyropod env
        is stepped (with its fused auto-reset), then one ``base_velocity_post`` launch dead-reckons (x, y) along the
        post-step yaw and carries out ``UpkieBaseVelocity.reset`` for the envs that reset in this tick. In next-step
        mode the MPC of a reset step runs on the terminal spine observation; the reset discards its result."""
        n = self.num_envs
        action = action.contiguous()
        self.sim._check_tensor(action, (n, 2), name="action")
        if self._spine is None:
            self._spine = self.sim.spine_obs()
        linear_velocity = action[:, 0].contiguous()
        ground_velocity = self.mpc_balancer.step_spine(linear_velocity, self._spine, self.dt)
        gyro_action = torch.stack([ground_velocity, action[:, 1]], dim=1).contiguous()
        fin6 = None
        if fin is not None:
            fin6 = getattr(self, "_gyro_final_obs", None)
            if fin6 is None:
                fin6 = self._gyro_final_obs = torch.zeros((n, 6), dtype=torch.float32, device=self.sim.device)
        # same-step mode: the resetting envs also stash their terminal state (info["final_info"])
        obs6, rew, term, trunc = self.sim.step_gyropod(gyro_action, final_obs=fin6, final_state=fin is not None)
        self._spine = self.sim.spine_obs()  # after a same-step reset: the reset's spine observation
        obs = torch.empty((n, 3), dtype=torch.float32, device=self.sim.device)  # a new tensor per step, as before
        base_velocity_post(self.sim, self.mpc_balancer, action, obs6, self._xy, self.dt, obs,
                           _AUTORESET[self.autoreset_mode], fin6, fin)
        self._bv_obs = obs
        return obs, rew, term, trunc

    def _device_final_obs(self) -> torch.Tensor:
        """Device final-observation rows of the same-step auto-reset, in the observation's layout (reused)."""
        fin = getattr(self, "_final_obs_tensor", None)
        if fin is None:
            shape = {"servos": (self.num_envs, 6, 5), "gyropod": (self.num_envs, 6), "pendulum": (self.num_envs, 4),
                     "base_velocity": (self.num_envs, 3)}
            fin = self._final_obs_tensor = torch.zeros(shape[self.env_type], dtype=torch.float32, device=self.sim.device)
        return fin
