# SPDX-License-Identifier: Apache-2.0
"""Tensor-level front end of the vectorised simulation (one handle = one GPU).

``UpkieSim`` owns a ``libupkie_b200`` handle and exposes the flat fast path of
SURVEY.md section 8(b): ``step_servos(action[N, 6, 6]) -> obs[N, 6, 5], reward[N],
terminated[N], truncated[N]`` over PyTorch CUDA tensors (PyTorch is used for
device memory and streams only; all arithmetic happens in the sm_90a kernels).
"""

import ctypes as C
from typing import Optional, Sequence, Tuple

import numpy as np
import torch

from . import _abi
from ._lib import check, lib
from .exceptions import UpkieException, UpkieRuntimeError
from .model import Model, default_model

AUTORESET_DISABLED, AUTORESET_NEXT_STEP, AUTORESET_SAME_STEP = 0, 1, 2


def _ptr(t: Optional[torch.Tensor]):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def _addr(x) -> Optional[int]:
    """Address of a tensor or ndarray for an ``UpkieStepOutputs`` field (None stays NULL)."""
    if x is None:
        return None
    return x.data_ptr() if isinstance(x, torch.Tensor) else x.ctypes.data


class UpkieSim:
    """N independent robots on one CUDA device.

    Replaces ``PyBulletBackend`` (``upkie/envs/backends/pybullet_backend.py:31``)
    for N robots at once; same constructor knobs (``dt``, ``nb_substeps``,
    ``torque_control_kp/kd``, ``joint_properties`` friction, ``inertia_variation``)
    through ``config`` / ``set_randomization``.
    """

    def __init__(
        self,
        n_envs: int,
        model: Optional[Model] = None,
        config: Optional[_abi.UpkieSimConfig] = None,
        device: int = 0,
    ):
        if not torch.cuda.is_available():
            raise UpkieRuntimeError(
                "upkie_b200 needs a CUDA device (there is no CPU fallback)"
            )
        self.model = model if model is not None else default_model()
        self.config = config if config is not None else _abi.default_sim_config()
        self.n = int(n_envs)
        self.device_index = int(device)
        self.device = torch.device("cuda", self.device_index)
        self._model_struct = self.model.to_struct()
        self._h = C.c_void_p()
        check(
            lib().upkie_b200_create(
                C.byref(self._model_struct), C.byref(self.config), self.n, self.device_index, C.byref(self._h)
            )
        )
        f32, u8 = torch.float32, torch.uint8
        dev = self.device
        self.reward = torch.empty(self.n, dtype=f32, device=dev)
        self.terminated = torch.empty(self.n, dtype=u8, device=dev)
        self.truncated = torch.empty(self.n, dtype=u8, device=dev)
        self.obs_servos = torch.empty((self.n, 6, 5), dtype=f32, device=dev)
        self.obs_gyropod = torch.empty((self.n, 6), dtype=f32, device=dev)
        self.obs_pendulum = torch.empty((self.n, 4), dtype=f32, device=dev)

    # ------------------------------------------------------------------
    def close(self) -> None:
        if getattr(self, "_h", None) is not None and self._h.value:
            lib().upkie_b200_destroy(self._h)
            self._h = C.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _stream(self):
        return C.c_void_p(torch.cuda.current_stream(self.device).cuda_stream)

    def _check_tensor(self, t: torch.Tensor, shape, dtype=torch.float32, name="tensor"):
        if t.device != self.device or t.dtype != dtype or not t.is_contiguous() or tuple(t.shape) != tuple(shape):
            raise UpkieRuntimeError(
                f"{name}: expected contiguous {dtype} tensor of shape {tuple(shape)} on {self.device}, "
                f"got {t.dtype} {tuple(t.shape)} on {t.device}"
            )

    # ------------------------------------------------------------------
    def set_autoreset(self, mode: int, seed: int = 0, env_offset: int = 0) -> None:
        check(lib().upkie_b200_set_autoreset(self._h, int(mode), int(seed), int(env_offset)))
        self._autoreset = (int(mode), int(seed), int(env_offset))

    def set_config(self, config: _abi.UpkieSimConfig) -> None:
        """Replace the configuration of the live handle (``upkie_b200_set_config``): initial-state bounds of the
        on-device reset sampler, noise levels, gains. Steps enqueued afterwards use it."""
        check(lib().upkie_b200_set_config(self._h, C.byref(config)))
        self.config = config

    def set_randomization(self, friction: Optional[torch.Tensor] = None, inertia_eps: Optional[torch.Tensor] = None):
        """Per-env floor friction [N] and ``randomize_inertias`` epsilons [N, 6]
        (``pybullet_backend.py:571-601``)."""
        if friction is not None:
            self._check_tensor(friction, (self.n,), name="friction")
        if inertia_eps is not None:
            self._check_tensor(inertia_eps, (self.n, 6), name="inertia_eps")
        check(lib().upkie_b200_set_randomization(self._h, _ptr(friction), _ptr(inertia_eps), self._stream()))
        torch.cuda.current_stream(self.device).synchronize()
        self._randomization = (None if friction is None else friction.clone(), None if inertia_eps is None else inertia_eps.clone())

    def set_env_params(self, rows: Optional[torch.Tensor] = None) -> None:
        """Per-env actuator and IMU parameters ``rows[N, EP_DIM]`` (layout ``_abi.EP_*``): env ``i`` runs
        ``torque_control_kp`` / ``kd``, joint friction, torque control / measurement noise and IMU uncertainty of row
        ``i`` instead of the config's, from the next step on. What N reference envs built with different
        ``PyBulletBackend`` arguments hold. ``None`` drops the table (every env runs the config's values again).
        Values must be finite, gains, friction and noise standard deviations >= 0; otherwise the call raises and the
        previous table stays."""
        if rows is not None:
            self._check_tensor(rows, (self.n, _abi.EP_DIM), name="env_params")
        check(lib().upkie_b200_set_env_params(self._h, _ptr(rows), self._stream()))
        self._env_params = None if rows is None else rows.clone()

    def get_env_params(self) -> torch.Tensor:
        """The parameters in force, ``[N, EP_DIM]``: the table, or without one the config's values in every row."""
        out = torch.empty((self.n, _abi.EP_DIM), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_env_params(self._h, _ptr(out), self._stream()))
        return out

    def get_randomization(self):
        """The randomisation in force: ``(friction[N], inertia_eps[N, 6])``, the nominal values where none is set."""
        friction = torch.empty(self.n, dtype=torch.float32, device=self.device)
        eps = torch.empty((self.n, 6), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_randomization(self._h, _ptr(friction), _ptr(eps), self._stream()))
        return friction, eps

    def set_reset_randomization(self, spec: Optional[_abi.UpkieResetRandomization]) -> None:
        """While ``spec`` is set, every reset of an env (fused auto-resets and ``reset``) redraws its selected columns
        uniformly from their ranges, keyed on the auto-reset seed, the global env index and the env's draw counter
        (``include/upkie_b200.h``). ``None`` turns it off; the values in force stay."""
        check(lib().upkie_b200_set_reset_randomization(self._h, C.byref(spec) if spec is not None else None))
        self._reset_randomization = None if spec is None else _abi.UpkieResetRandomization.from_buffer_copy(spec)
        if spec is not None:
            self._randomized_at_reset = True  # the values in force are no longer the ones last set from the host

    def get_draws(self) -> torch.Tensor:
        """Per-env draw counters of the reset randomisation ``[N]`` (int32 bits of uint32)."""
        out = torch.empty(self.n, dtype=torch.int32, device=self.device)
        check(lib().upkie_b200_get_draws(self._h, _ptr(out), self._stream()))
        return out

    def set_draws(self, draws: torch.Tensor) -> None:
        self._check_tensor(draws, (self.n,), torch.int32, "draws")
        check(lib().upkie_b200_set_draws(self._h, _ptr(draws), self._stream()))

    def set_push_randomization(self, spec: Optional[_abi.UpkiePushRandomization]) -> None:
        """While ``spec`` is set, every env is pushed on one body by random world-frame forces at random times, drawn
        and applied by the step kernel: after each reset, ``gap`` steps without a push, ``duration`` steps of a
        constant force, then the next draw (``include/upkie_b200.h``). ``None`` turns it off; no counter restarts."""
        check(lib().upkie_b200_set_push_randomization(self._h, C.byref(spec) if spec is not None else None))
        self._push_randomization = None if spec is None else _abi.UpkiePushRandomization.from_buffer_copy(spec)

    def get_push_forces(self) -> torch.Tensor:
        """The push force ``[N, 3]`` (world frame, N) applied in each env's last step; zero where none was."""
        out = torch.empty((self.n, 3), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_push_forces(self._h, _ptr(out), self._stream()))
        return out

    def get_push_state(self):
        """Per-env push schedule state ``(count[N], timer[N])`` (int32 bits of uint32)."""
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        timer = torch.empty(self.n, dtype=torch.int32, device=self.device)
        check(lib().upkie_b200_get_push_state(self._h, _ptr(count), _ptr(timer), self._stream()))
        return count, timer

    def set_push_state(self, count: torch.Tensor, timer: torch.Tensor) -> None:
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(timer, (self.n,), torch.int32, "timer")
        check(lib().upkie_b200_set_push_state(self._h, _ptr(count), _ptr(timer), self._stream()))

    def set_action_delay(self, low: Optional[int], high: Optional[int] = None, max_ticks: int = 1) -> None:
        """While a range is set, every env applies its servo command ``d`` substeps into each tick, ``low <= d <= high
        <= nb_substeps``: the substeps before ``d`` run the command of its previous tick. Each reset of the env draws a
        new ``d`` (keyed on the auto-reset seed and the env's counter, ``include/upkie_b200.h``) and stops the servos
        until the first command takes over. ``high`` defaults to ``low``; ``None`` turns the delay off. Setting a range
        draws nothing: it takes effect at each env's next reset.

        ``max_ticks`` (1 .. ``MAX_DELAY_TICKS``) is the history of commands each env keeps, in ticks: ``high`` may then
        reach ``max_ticks * nb_substeps``, and a delay ``d = q * nb_substeps + r`` (``1 <= r <= nb_substeps``) runs the
        command of ``q`` ticks earlier from substep ``r`` on and the one before it until then. A change of depth keeps
        the history in age order, truncated or extended with stop rows."""
        if low is None:
            check(lib().upkie_b200_set_action_delay(self._h, None))
            self._action_delay = None
            return
        spec = _abi.UpkieActionDelay(int(low), int(low if high is None else high))
        check(lib().upkie_b200_set_action_delay_ticks(self._h, C.byref(spec), int(max_ticks)))
        self._action_delay = (spec.substeps_low, spec.substeps_high)
        self._action_delay_ticks = int(max_ticks)
        self._delay_state_set = True  # the handle holds a state from now on

    def get_action_delay_history(self) -> torch.Tensor:
        """``[max_ticks, N, 6, 6]`` the servo commands of each env's last ``max_ticks`` ticks, the newest first (stop
        rows before the env's last reset)."""
        out = torch.empty((getattr(self, "_action_delay_ticks", 1), self.n, _abi.NJ, len(_abi.ACT_KEYS)),
                          dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_action_delay_history(self._h, _ptr(out), self._stream()))
        return out

    def set_action_delay_history(self, commands: torch.Tensor) -> None:
        self._check_tensor(commands, (getattr(self, "_action_delay_ticks", 1), self.n, _abi.NJ, len(_abi.ACT_KEYS)),
                           name="commands")
        check(lib().upkie_b200_set_action_delay_history(self._h, _ptr(commands), self._stream()))
        self._delay_state_set = True

    def get_action_delay_state(self):
        """Per-env action-delay state ``(count[N], delay[N], command[N, 6, 6])``: the draw counters (int32 bits of
        uint32), the delays in substeps and the servo command of each env's previous tick."""
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        delay = torch.empty(self.n, dtype=torch.int32, device=self.device)
        command = torch.empty((self.n, _abi.NJ, len(_abi.ACT_KEYS)), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_action_delay_state(self._h, _ptr(count), _ptr(delay), _ptr(command),
                                                      self._stream()))
        return count, delay, command

    def set_action_delay_state(self, count: torch.Tensor, delay: torch.Tensor, command: torch.Tensor) -> None:
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(delay, (self.n,), torch.int32, "delay")
        self._check_tensor(command, (self.n, _abi.NJ, len(_abi.ACT_KEYS)), name="command")
        check(lib().upkie_b200_set_action_delay_state(self._h, _ptr(count), _ptr(delay), _ptr(command),
                                                      self._stream()))
        self._delay_state_set = True

    def set_observation_delay(self, low: Optional[int], high: Optional[int] = None, max_ticks: int = 1) -> None:
        """While a range is set, everything a step reports about each env's sensors (its observation, ``spine_obs``,
        ``final_obs`` and the final spine observation) describes the robot ``d`` substeps before the end of the tick,
        ``low <= d <= high <= nb_substeps``; the IMU acceleration differentiates consecutive snapshots. Terminations,
        resets and ``get_state`` read the true state. Each reset of the env draws a new ``d`` (keyed on the auto-reset
        seed and the env's counter, ``include/upkie_b200.h``) and is observed undelayed. ``high`` defaults to ``low``;
        ``None`` turns the delay off. Setting a range draws nothing: it takes effect at each env's next reset.

        ``max_ticks`` (1 .. ``MAX_DELAY_TICKS``) is the history of snapshots each env keeps, in ticks: ``high`` may then
        reach ``max_ticks * nb_substeps``, and a delay ``d = q * nb_substeps + r`` (``1 <= r <= nb_substeps``) reports
        what a delay of ``r`` reported ``q`` ticks earlier, the post-reset state for the ticks before the env's last
        reset. A change of depth keeps the history in age order, truncated or extended with copies of the oldest."""
        if low is None:
            check(lib().upkie_b200_set_observation_delay(self._h, None))
            self._observation_delay = None
            return
        spec = _abi.UpkieObservationDelay(int(low), int(low if high is None else high))
        check(lib().upkie_b200_set_observation_delay_ticks(self._h, C.byref(spec), int(max_ticks)))
        self._observation_delay = (spec.substeps_low, spec.substeps_high)
        self._observation_delay_ticks = int(max_ticks)
        self._sense_state_set = True  # the handle holds a state from now on

    def get_observation_delay_history(self) -> torch.Tensor:
        """``[max_ticks, N, STATE_DIM]`` the sensor snapshots of each env's last ``max_ticks`` ticks, the newest first
        (``get_state`` layout, the sensed columns; the post-reset state before the env's last reset). At depth 1 the
        sensed rows of ``get_observation_delay_state``."""
        out = torch.empty((getattr(self, "_observation_delay_ticks", 1), self.n, _abi.STATE_DIM), dtype=torch.float32,
                          device=self.device)
        check(lib().upkie_b200_get_observation_delay_history(self._h, _ptr(out), self._stream()))
        return out

    def set_observation_delay_history(self, rows: torch.Tensor) -> None:
        self._check_tensor(rows, (getattr(self, "_observation_delay_ticks", 1), self.n, _abi.STATE_DIM), name="rows")
        check(lib().upkie_b200_set_observation_delay_history(self._h, _ptr(rows), self._stream()))
        self._sense_state_set = True

    def get_observation_delay_state(self):
        """Per-env observation-delay state ``(count[N], delay[N], rows[N, STATE_DIM])``: the draw counters (int32 bits
        of uint32), the delays in substeps and the sensed state rows (``get_state`` layout), what the observations are
        built from; the current state on a handle that never had a delay."""
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        delay = torch.empty(self.n, dtype=torch.int32, device=self.device)
        rows = torch.empty((self.n, _abi.STATE_DIM), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_observation_delay_state(self._h, _ptr(count), _ptr(delay), _ptr(rows),
                                                           self._stream()))
        return count, delay, rows

    def set_observation_delay_state(self, count: torch.Tensor, delay: torch.Tensor, rows: torch.Tensor) -> None:
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(delay, (self.n,), torch.int32, "delay")
        self._check_tensor(rows, (self.n, _abi.STATE_DIM), name="rows")
        check(lib().upkie_b200_set_observation_delay_state(self._h, _ptr(count), _ptr(delay), _ptr(rows),
                                                           self._stream()))
        self._sense_state_set = True

    def set_servo_dropout(self, low: Optional[float], high: Optional[float] = None,
                          joints: Optional[Sequence[str]] = None) -> None:
        """While a range is set, each reply of the servos ``joints`` (names, None: all six) is lost in each substep (a
        1 kHz spine cycle) with each env's probability ``p ~ U(low, high)``, drawn at every reset of the env (keyed on
        the auto-reset seed and the env's counter, ``include/upkie_b200.h``). A servo whose reply is lost reports the
        position, velocity and torque of its last received reply in every observation, ``spine_obs`` (its wheel
        odometry too), the final observations and the history; the physics, terminations and ``get_state`` see the
        true state. ``high`` defaults to ``low``; ``None`` turns the dropouts off. Setting a range draws nothing: it
        takes effect at each env's next reset."""
        if low is None:
            check(lib().upkie_b200_set_servo_dropout(self._h, None))
            self._servo_dropout = None
            return
        names = _abi.JOINT_NAMES if joints is None else list(joints)
        unknown = [j for j in names if j not in _abi.JOINT_NAMES]
        if unknown:
            raise UpkieException(f"set_servo_dropout: unknown joint(s) {unknown}")
        mask = sum(1 << _abi.JOINT_NAMES.index(j) for j in set(names))
        spec = _abi.UpkieServoDropout(float(low), float(low if high is None else high), mask, 0)
        check(lib().upkie_b200_set_servo_dropout(self._h, C.byref(spec)))
        self._servo_dropout = (spec.prob_low, spec.prob_high, mask)

    @property
    def servo_dropout_spec(self) -> Optional[Tuple[float, float, int]]:
        """``(prob_low, prob_high, joint_mask)`` of the servo dropouts in force, or None."""
        return getattr(self, "_servo_dropout", None)

    def get_servo_dropout_state(self):
        """Per-env servo-dropout state ``(count[N], prob[N], held[N, 6, 3])``: the draw counters (int32 bits of
        uint32), the loss probabilities and the latched ``[joint][position, velocity, torque]``."""
        if self.servo_dropout_spec is None:
            raise UpkieException("no servo dropouts are set (set_servo_dropout)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        prob = torch.empty(self.n, dtype=torch.float32, device=self.device)
        held = torch.empty((self.n, _abi.NJ, 3), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_servo_dropout_state(self._h, _ptr(count), _ptr(prob), _ptr(held), self._stream()))
        return count, prob, held

    def set_servo_dropout_state(self, count: torch.Tensor, prob: torch.Tensor, held: torch.Tensor) -> None:
        if self.servo_dropout_spec is None:
            raise UpkieException("no servo dropouts are set (set_servo_dropout)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(prob, (self.n,), name="prob")
        self._check_tensor(held, (self.n, _abi.NJ, 3), name="held")
        check(lib().upkie_b200_set_servo_dropout_state(self._h, _ptr(count), _ptr(prob), _ptr(held), self._stream()))

    def set_imu_misalignment(self, roll: Optional[Tuple[float, float]] = (0.0, 0.0),
                             pitch: Tuple[float, float] = (0.0, 0.0), yaw: Tuple[float, float] = (0.0, 0.0)) -> None:
        """While ranges are set, each env's IMU is mounted off its nominal pose by E = Rz(yaw) Ry(pitch) Rx(roll), the
        three angles (radians) drawn from ``(low, high)`` ranges at every reset of the env (keyed on the auto-reset seed
        and the env's counter, ``include/upkie_b200.h``). Every orientation-derived observation (base pitch, angular
        velocity and rotation, the IMU orientation, rates and accelerations, the gyropod and pendulum pitch and rate)
        is that of a base oriented R E instead of R; the physics, terminations and ``get_state`` see the true state.
        ``roll=None`` turns the misalignment off. Setting ranges draws nothing: they take effect at each env's next
        reset."""
        if roll is None:
            check(lib().upkie_b200_set_imu_misalignment(self._h, None))
            self._imu_misalignment = None
            return
        spec = _abi.UpkieImuMisalignment(*(float(v) for r in (roll, pitch, yaw) for v in r))
        check(lib().upkie_b200_set_imu_misalignment(self._h, C.byref(spec)))
        self._imu_misalignment = ((spec.roll_low, spec.roll_high), (spec.pitch_low, spec.pitch_high),
                                  (spec.yaw_low, spec.yaw_high))

    @property
    def imu_misalignment_spec(self) -> Optional[Tuple[Tuple[float, float], ...]]:
        """``((roll_low, roll_high), (pitch_low, pitch_high), (yaw_low, yaw_high))`` in force, or None."""
        return getattr(self, "_imu_misalignment", None)

    def get_imu_misalignment_state(self):
        """Per-env IMU-misalignment state ``(count[N], quat[N, 4])``: the draw counters (int32 bits of uint32) and each
        env's misalignment as a unit quaternion (w, x, y, z)."""
        if self.imu_misalignment_spec is None:
            raise UpkieException("no IMU misalignment is set (set_imu_misalignment)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        quat = torch.empty((self.n, 4), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_imu_misalignment_state(self._h, _ptr(count), _ptr(quat), self._stream()))
        return count, quat

    def set_imu_misalignment_state(self, count: torch.Tensor, quat: torch.Tensor) -> None:
        """Set every env's draw counter and misalignment quaternion (w, x, y, z), unit within 1e-5: a checkpoint, or
        fixed offsets of the caller's choice (kept until each env's next reset)."""
        if self.imu_misalignment_spec is None:
            raise UpkieException("no IMU misalignment is set (set_imu_misalignment)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(quat, (self.n, 4), name="quat")
        check(lib().upkie_b200_set_imu_misalignment_state(self._h, _ptr(count), _ptr(quat), self._stream()))

    def set_attitude_filter(self, kp: Optional[Tuple[float, float]], ki: Tuple[float, float] = (0.0, 0.0),
                            roll: Tuple[float, float] = (0.0, 0.0), pitch: Tuple[float, float] = (0.0, 0.0)) -> None:
        """While ranges are set, each env runs an attitude filter on its simulated IMU (an explicit complementary filter
        with gyro-bias estimation, once per substep; ``include/upkie_b200.h``), and every orientation-derived
        observation (the IMU orientation, the base pitch and ``rotation_base_to_world``, the gyropod and pendulum
        pitch) reports its estimate instead of the true orientation; the rates, accelerations, physics, terminations
        and ``get_state`` are untouched. Every reset of an env draws its gains ``kp`` (1/s) and ``ki`` (1/s^2) and an
        initial estimate error ``roll``, ``pitch`` (rad, about the base axes) from ``(low, high)`` ranges, keyed on the
        auto-reset seed and the env's counter. ``kp=None`` turns the filter off. Setting ranges draws nothing: an env
        of a handle without a filter starts from the true orientation with the upper gains until its next reset."""
        if kp is None:
            check(lib().upkie_b200_set_attitude_filter(self._h, None))
            self._attitude_filter = None
            return
        spec = _abi.UpkieAttitudeFilter(*(float(v) for r in (kp, ki, roll, pitch) for v in r))
        check(lib().upkie_b200_set_attitude_filter(self._h, C.byref(spec)))
        self._attitude_filter = ((spec.kp_low, spec.kp_high), (spec.ki_low, spec.ki_high),
                                 (spec.roll_low, spec.roll_high), (spec.pitch_low, spec.pitch_high))

    @property
    def attitude_filter_spec(self) -> Optional[Tuple[Tuple[float, float], ...]]:
        """``((kp_low, kp_high), (ki_low, ki_high), (roll_low, roll_high), (pitch_low, pitch_high))`` in force, or
        None."""
        return getattr(self, "_attitude_filter", None)

    def get_attitude_filter_state(self):
        """Per-env attitude-filter state ``(count[N], gains[N, 2], quat[N, 4], bias[N, 3])``: the draw counters (int32
        bits of uint32), the gains (kp, ki), the estimated IMU-to-world rotation (w, x, y, z) and the gyro-bias
        estimate (rad/s, IMU frame)."""
        if self.attitude_filter_spec is None:
            raise UpkieException("no attitude filter is set (set_attitude_filter)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        gains = torch.empty((self.n, 2), dtype=torch.float32, device=self.device)
        quat = torch.empty((self.n, 4), dtype=torch.float32, device=self.device)
        bias = torch.empty((self.n, 3), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_attitude_filter_state(self._h, _ptr(count), _ptr(gains), _ptr(quat), _ptr(bias),
                                                         self._stream()))
        return count, gains, quat, bias

    def set_attitude_filter_state(self, count: torch.Tensor, gains: torch.Tensor, quat: torch.Tensor,
                                  bias: torch.Tensor) -> None:
        """Set every env's draw counter, gains, estimate (unit within 1e-5) and bias estimate: a checkpoint."""
        if self.attitude_filter_spec is None:
            raise UpkieException("no attitude filter is set (set_attitude_filter)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(gains, (self.n, 2), name="gains")
        self._check_tensor(quat, (self.n, 4), name="quat")
        self._check_tensor(bias, (self.n, 3), name="bias")
        check(lib().upkie_b200_set_attitude_filter_state(self._h, _ptr(count), _ptr(gains), _ptr(quat), _ptr(bias),
                                                         self._stream()))

    def get_attitude_filter_report(self) -> torch.Tensor:
        """``[N, 4]`` the estimate (w, x, y, z, IMU to world) each env's observation reports under an observation delay:
        that of the cycle its snapshot observed."""
        if self.attitude_filter_spec is None:
            raise UpkieException("no attitude filter is set (set_attitude_filter)")
        out = torch.empty((self.n, 4), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_attitude_filter_report(self._h, _ptr(out), self._stream()))
        return out

    def set_attitude_filter_report(self, quat: torch.Tensor) -> None:
        """Set every env's reported estimate (unit within 1e-5, see ``get_attitude_filter_report``): a checkpoint.
        ``set_attitude_filter_state`` leaves it, as setting the estimate leaves an observation delay's snapshot."""
        if self.attitude_filter_spec is None:
            raise UpkieException("no attitude filter is set (set_attitude_filter)")
        self._check_tensor(quat, (self.n, 4), name="quat")
        check(lib().upkie_b200_set_attitude_filter_report(self._h, _ptr(quat), self._stream()))

    def set_encoder_offset(self, low: Optional[float], high: Optional[float] = None,
                           joints: Optional[Sequence[str]] = None) -> None:
        """While a range is set, each servo of ``joints`` (names, None: the four hip and knee joints) is zeroed off by
        an offset ``delta ~ U(low, high)`` radians, drawn per joint at every reset of the env (keyed on the auto-reset
        seed and the env's counter, ``include/upkie_b200.h``). The servo frame is the joint frame shifted by delta:
        every reported position (the servo rows, ``spine_obs`` and its wheel odometry, the gyropod and pendulum ``p``,
        the final observations and the history) is ``q + delta``, every position target executes as ``target - delta``,
        and the gyropod, pendulum and base-velocity leg targets are servo-frame values (a reset sets them to the
        reported positions). The physics, terminations and ``get_state``'s q see the true joints. ``high`` defaults to
        ``low``; ``None`` turns the offsets off. Setting a range draws nothing: it takes effect at each env's next
        reset."""
        if low is None:
            check(lib().upkie_b200_set_encoder_offset(self._h, None))
            self._encoder_offset = None
            return
        names = list(_abi.ENCODER_OFFSET_DEFAULT_JOINTS) if joints is None else list(joints)
        unknown = [j for j in names if j not in _abi.JOINT_NAMES]
        if unknown:
            raise UpkieException(f"set_encoder_offset: unknown joint(s) {unknown}")
        mask = sum(1 << _abi.JOINT_NAMES.index(j) for j in set(names))
        spec = _abi.UpkieEncoderOffset(float(low), float(low if high is None else high), mask, 0)
        check(lib().upkie_b200_set_encoder_offset(self._h, C.byref(spec)))
        self._encoder_offset = (spec.low, spec.high, mask)

    @property
    def encoder_offset_spec(self) -> Optional[Tuple[float, float, int]]:
        """``(low, high, joint_mask)`` of the encoder offsets in force, or None."""
        return getattr(self, "_encoder_offset", None)

    def get_encoder_offset_state(self):
        """Per-env encoder-offset state ``(count[N], offset[N, 6])``: the draw counters (int32 bits of uint32) and each
        env's zero offset per joint, in radians."""
        if self.encoder_offset_spec is None:
            raise UpkieException("no encoder offsets are set (set_encoder_offset)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        offset = torch.empty((self.n, _abi.NJ), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_encoder_offset_state(self._h, _ptr(count), _ptr(offset), self._stream()))
        return count, offset

    def set_encoder_offset_state(self, count: torch.Tensor, offset: torch.Tensor) -> None:
        """Set every env's draw counter and zero offsets (finite, within 0.5 rad, zero outside the mask): a checkpoint,
        or offsets measured on a robot (kept until each env's next reset)."""
        if self.encoder_offset_spec is None:
            raise UpkieException("no encoder offsets are set (set_encoder_offset)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(offset, (self.n, _abi.NJ), name="offset")
        check(lib().upkie_b200_set_encoder_offset_state(self._h, _ptr(count), _ptr(offset), self._stream()))

    def set_servo_noise(self, position=None, velocity=None) -> None:
        """While ranges are set, every reported servo position and velocity carries white noise: each reset of an env
        draws one standard deviation per joint and quantity, ``sigma ~ U(low, high)`` (radians for ``position``, rad/s
        for ``velocity``, each a ``(low[6], high[6])`` pair in ``JOINT_NAMES`` order; None: no noise on that quantity),
        and each spine cycle adds ``sigma * n``, n a standard normal keyed on the auto-reset seed, the env and the
        cycle (``include/upkie_b200.h``). Every output that reports a cycle reports the same noise: the servo rows,
        ``spine_obs`` and its wheel odometry, the gyropod and pendulum ``p`` / ``pdot``, the final observations and the
        history. The physics, the torques and ``get_state`` see the true replies. Both None turns the noise off.
        Setting ranges draws nothing: they take effect at each env's next reset."""
        if position is None and velocity is None:
            check(lib().upkie_b200_set_servo_noise(self._h, None))
            self._servo_noise = None
            return
        spec = _abi.UpkieServoNoise()
        for name, pair in (("position", position), ("velocity", velocity)):
            lo, hi = ([0.0] * _abi.NJ, [0.0] * _abi.NJ) if pair is None else pair
            lo = np.asarray(lo, dtype=np.float32).reshape(-1)
            hi = np.asarray(hi, dtype=np.float32).reshape(-1)
            if lo.shape != (_abi.NJ,) or hi.shape != (_abi.NJ,):
                raise UpkieException(f"set_servo_noise: {name} expects (low[6], high[6])")
            getattr(spec, f"{name}_low")[:] = [float(x) for x in lo]
            getattr(spec, f"{name}_high")[:] = [float(x) for x in hi]
        check(lib().upkie_b200_set_servo_noise(self._h, C.byref(spec)))
        self._servo_noise = ((tuple(spec.position_low), tuple(spec.position_high)),
                             (tuple(spec.velocity_low), tuple(spec.velocity_high)))

    @property
    def servo_noise_spec(self):
        """``((position_low, position_high), (velocity_low, velocity_high))`` of the servo noise in force, or None."""
        return getattr(self, "_servo_noise", None)

    def get_servo_noise_state(self):
        """Per-env servo-noise state ``(count[N], sigma[N, 12])``: the draw counters (int32 bits of uint32) and each
        env's standard deviations, columns 0-5 the joints' position noise (rad), 6-11 their velocity noise (rad/s)."""
        if self.servo_noise_spec is None:
            raise UpkieException("no servo noise is set (set_servo_noise)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        sigma = torch.empty((self.n, 2 * _abi.NJ), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_servo_noise_state(self._h, _ptr(count), _ptr(sigma), self._stream()))
        return count, sigma

    def set_servo_noise_state(self, count: torch.Tensor, sigma: torch.Tensor) -> None:
        """Set every env's draw counter and standard deviations (finite, >= 0, at most 0.1 rad / 5 rad/s, zero in a
        column whose high bound is zero): a checkpoint, or levels measured on a robot (kept until each env's next
        reset)."""
        if self.servo_noise_spec is None:
            raise UpkieException("no servo noise is set (set_servo_noise)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(sigma, (self.n, 2 * _abi.NJ), name="sigma")
        check(lib().upkie_b200_set_servo_noise_state(self._h, _ptr(count), _ptr(sigma), self._stream()))

    def set_velocity_derate(self, max_velocity=None, derate=None, joints: Optional[Sequence[str]] = None) -> None:
        """While limits are set, each servo of ``joints`` (names, None: all six) derates its torque past a velocity
        limit, as the moteus ``servo.max_velocity`` does: every reset of an env draws one limit per joint,
        ``v ~ U(low, high)`` in rad/s (keyed on the auto-reset seed and the env's counter, ``include/upkie_b200.h``),
        and in every substep a joint with ``|qd| > v`` has the torque that drives it faster capped by
        ``clip((v + derate - |qd|) / derate, 0, 1) * tau_max``; a braking torque passes unchanged. A speed in rev/s is
        ``2 * pi`` times that in rad/s: the robot's 2 rev/s is 12.57 rad/s. ``max_velocity`` is a ``(low, high)`` pair of
        bounds or a sequence of six per-joint ``(low, high)`` pairs (``JOINT_NAMES`` order), ``derate`` a band in
        rad/s or six of them (None: ``MOTEUS_MAX_VELOCITY_DERATE``, 2 rev/s); ``max_velocity=None`` turns the limits
        off. Setting limits draws nothing: each env keeps
        the limits of the joints that stay limited until its next reset, and the joints a spec adds take ``high``
        until then."""
        if max_velocity is None:
            check(lib().upkie_b200_set_velocity_derate(self._h, None))
            self._velocity_derate = None
            return
        mv = np.asarray(max_velocity, dtype=np.float32)
        if mv.shape == (2,):
            lo, hi = np.full(_abi.NJ, mv[0], np.float32), np.full(_abi.NJ, mv[1], np.float32)
        elif mv.shape == (_abi.NJ, 2):
            lo, hi = mv[:, 0], mv[:, 1]
        else:
            raise UpkieException("set_velocity_derate: max_velocity expects (low, high) or six (low, high) pairs")
        d = np.asarray(_abi.MOTEUS_MAX_VELOCITY_DERATE if derate is None else derate, dtype=np.float32).reshape(-1)
        if d.shape == (1,):
            d = np.repeat(d, _abi.NJ)
        if d.shape != (_abi.NJ,):
            raise UpkieException("set_velocity_derate: derate expects one band or six")
        names = list(_abi.JOINT_NAMES) if joints is None else list(joints)
        unknown = [j for j in names if j not in _abi.JOINT_NAMES]
        if unknown:
            raise UpkieException(f"set_velocity_derate: unknown joint(s) {unknown}")
        mask = sum(1 << _abi.JOINT_NAMES.index(j) for j in set(names))
        spec = _abi.UpkieVelocityDerate()
        spec.max_velocity_low[:] = [float(x) for x in lo]
        spec.max_velocity_high[:] = [float(x) for x in hi]
        spec.derate[:] = [float(x) for x in d]
        spec.joint_mask = mask
        check(lib().upkie_b200_set_velocity_derate(self._h, C.byref(spec)))
        self._velocity_derate = (tuple(zip(spec.max_velocity_low, spec.max_velocity_high)), tuple(spec.derate), mask)

    @property
    def velocity_derate_spec(self):
        """``(max_velocity, derate, joint_mask)`` of the velocity limits in force (six ``(low, high)`` pairs and six
        bands, rad/s), or None."""
        return getattr(self, "_velocity_derate", None)

    def get_velocity_derate_state(self):
        """Per-env velocity-limit state ``(count[N], max_velocity[N, 6])``: the draw counters (int32 bits of uint32)
        and each env's limit per joint in rad/s (0 for a joint without one)."""
        if self.velocity_derate_spec is None:
            raise UpkieException("no velocity limits are set (set_velocity_derate)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        vmax = torch.empty((self.n, _abi.NJ), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_velocity_derate_state(self._h, _ptr(count), _ptr(vmax), self._stream()))
        return count, vmax

    def set_velocity_derate_state(self, count: torch.Tensor, max_velocity: torch.Tensor) -> None:
        """Set every env's draw counter and velocity limits (finite and > 0 on a limited joint, zero on the others): a
        checkpoint, or limits configured on a robot (kept until each env's next reset)."""
        if self.velocity_derate_spec is None:
            raise UpkieException("no velocity limits are set (set_velocity_derate)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(max_velocity, (self.n, _abi.NJ), name="max_velocity")
        check(lib().upkie_b200_set_velocity_derate_state(self._h, _ptr(count), _ptr(max_velocity), self._stream()))

    def set_torque_scale(self, scale=None, joints: Optional[Sequence[str]] = None) -> None:
        """While scales are set, each joint of ``joints`` (names, None: all six) receives a scale of the torque its servo
        commands and reports, as a servo whose torque constant is off: every reset of an env draws one scale per joint,
        ``s ~ U(low, high)`` (keyed on the auto-reset seed and the env's counter, ``include/upkie_b200.h``), and in every
        substep the physics integrates ``s * t`` for the servo's torque ``t`` (after its clip and velocity derate),
        while the torque replies and ``get_state`` keep ``t``. ``scale`` is a ``(low, high)`` pair of bounds or a
        sequence of six per-joint ``(low, high)`` pairs (``JOINT_NAMES`` order), with ``0 < low <= high <= 2``;
        ``(0.9, 1.1)`` is a usual "motor strength" range in legged-robot RL, not a measured figure of the Upkie's
        servos. ``scale=None`` turns the scales off. Setting scales draws nothing: each env keeps the scales of the
        joints that stay scaled until its next reset, and the joints a spec adds hold 1 until then."""
        if scale is None:
            check(lib().upkie_b200_set_torque_scale(self._h, None))
            self._torque_scale = None
            return
        sc = np.asarray(scale, dtype=np.float32)
        if sc.shape == (2,):
            lo, hi = np.full(_abi.NJ, sc[0], np.float32), np.full(_abi.NJ, sc[1], np.float32)
        elif sc.shape == (_abi.NJ, 2):
            lo, hi = sc[:, 0], sc[:, 1]
        else:
            raise UpkieException("set_torque_scale: scale expects (low, high) or six (low, high) pairs")
        names = list(_abi.JOINT_NAMES) if joints is None else list(joints)
        unknown = [j for j in names if j not in _abi.JOINT_NAMES]
        if unknown:
            raise UpkieException(f"set_torque_scale: unknown joint(s) {unknown}")
        mask = sum(1 << _abi.JOINT_NAMES.index(j) for j in set(names))
        spec = _abi.UpkieTorqueScale()
        spec.scale_low[:] = [float(x) for x in lo]
        spec.scale_high[:] = [float(x) for x in hi]
        spec.joint_mask = mask
        check(lib().upkie_b200_set_torque_scale(self._h, C.byref(spec)))
        self._torque_scale = (tuple(zip(spec.scale_low, spec.scale_high)), mask)

    @property
    def torque_scale_spec(self):
        """``(scale, joint_mask)`` of the torque scales in force (six ``(low, high)`` pairs), or None."""
        return getattr(self, "_torque_scale", None)

    def get_torque_scale_state(self):
        """Per-env torque-scale state ``(count[N], scale[N, 6])``: the draw counters (int32 bits of uint32) and each
        env's scale per joint (exactly 1 for a joint without one)."""
        if self.torque_scale_spec is None:
            raise UpkieException("no torque scales are set (set_torque_scale)")
        count = torch.empty(self.n, dtype=torch.int32, device=self.device)
        scale = torch.empty((self.n, _abi.NJ), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_torque_scale_state(self._h, _ptr(count), _ptr(scale), self._stream()))
        return count, scale

    def set_torque_scale_state(self, count: torch.Tensor, scale: torch.Tensor) -> None:
        """Set every env's draw counter and torque scales (in ``(0, 2]`` on a scaled joint, exactly 1 on the others): a
        checkpoint, or fixed scales (kept until each env's next reset)."""
        if self.torque_scale_spec is None:
            raise UpkieException("no torque scales are set (set_torque_scale)")
        self._check_tensor(count, (self.n,), torch.int32, "count")
        self._check_tensor(scale, (self.n, _abi.NJ), name="scale")
        check(lib().upkie_b200_set_torque_scale_state(self._h, _ptr(count), _ptr(scale), self._stream()))

    def get_servo_noise_mark(self) -> torch.Tensor:
        """Per-env mark ``[N]`` (uint8): 1 while the env reports its reset observation (``spine_obs`` and
        ``reset_obs`` then carry the reset cycle's noise), 0 after a step that did not reset it."""
        if self.servo_noise_spec is None:
            raise UpkieException("no servo noise is set (set_servo_noise)")
        mark = torch.empty(self.n, dtype=torch.uint8, device=self.device)
        check(lib().upkie_b200_get_servo_noise_mark(self._h, _ptr(mark), self._stream()))
        return mark

    def set_servo_noise_mark(self, mark: torch.Tensor) -> None:
        """Set every env's mark (0 or 1, see ``get_servo_noise_mark``): a checkpoint."""
        if self.servo_noise_spec is None:
            raise UpkieException("no servo noise is set (set_servo_noise)")
        self._check_tensor(mark, (self.n,), torch.uint8, "mark")
        check(lib().upkie_b200_set_servo_noise_mark(self._h, _ptr(mark), self._stream()))

    def set_history(self, columns: Optional[Sequence[int]], size: int = 1) -> None:
        """Record each env's spine-observation ``columns`` (``_abi.SP_*``, 1 to ``MAX_HISTORY_CHANNELS`` of them) after
        every substep, and report the last ``size`` (1 to ``MAX_HISTORY``) through ``get_history``: the spine's
        ``HistoryObserver`` (``upkie/cpp/observers/HistoryObserver.h``) at the substep rate. Entry 0 is the observed
        instant (the end of the tick, or the observation delay's snapshot), entry k is k substeps earlier. The IMU
        accelerations differentiate over one substep, the torques are the applied ones without measurement noise. Each
        reset of an env fills its entries with its post-reset columns; a new spec and ``set_state`` fill every env's.
        ``None`` turns it off. The history records only: every other output of a step is unchanged."""
        if columns is None:
            check(lib().upkie_b200_set_history(self._h, None))
            self._history = None
            return
        cols = [int(c) for c in columns]
        if not 1 <= len(cols) <= _abi.MAX_HISTORY_CHANNELS:
            raise UpkieException(f"set_history: 1 to {_abi.MAX_HISTORY_CHANNELS} columns, got {len(cols)}")
        spec = _abi.UpkieHistory(int(size), len(cols))
        for k, c in enumerate(cols):
            spec.columns[k] = c
        check(lib().upkie_b200_set_history(self._h, C.byref(spec)))
        self._history = (tuple(cols), int(size))

    @property
    def history_spec(self) -> Optional[Tuple[Tuple[int, ...], int]]:
        """``(columns, size)`` of the history in force, or None."""
        return getattr(self, "_history", None)

    def get_history(self) -> torch.Tensor:
        """``[N, size, C]`` the history's entries of every env, newest first (``set_history``)."""
        cols, size = self._require_history()
        out = torch.empty((self.n, size, len(cols)), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_history(self._h, _ptr(out), self._stream()))
        return out

    def _require_history(self):
        if self.history_spec is None:
            raise UpkieException("no observation history is set (set_history)")
        return self.history_spec

    def history_entries(self) -> int:
        """Entries of the history's ring: ``size`` plus the deepest observation delay, in substeps (0: no history)."""
        t = C.c_int(0)
        check(lib().upkie_b200_history_entries(self._h, C.byref(t)))
        return int(t.value)

    def get_history_state(self) -> torch.Tensor:
        """``[history_entries(), N, C]`` the whole ring in age order, 0 the entry the last substep wrote (checkpoints)."""
        cols, _ = self._require_history()
        out = torch.empty((self.history_entries(), self.n, len(cols)), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_history_state(self._h, _ptr(out), self._stream()))
        return out

    def set_history_state(self, rows: torch.Tensor) -> None:
        cols, _ = self._require_history()
        self._check_tensor(rows, (self.history_entries(), self.n, len(cols)), name="rows")
        check(lib().upkie_b200_set_history_state(self._h, _ptr(rows), self._stream()))

    def set_external_forces(self, force: Optional[torch.Tensor] = None, local_mask: int = 0) -> None:
        """``force[N, 7, 3]`` newtons at the centres of mass of the 7 bodies, applied on every substep of
        the following steps until overwritten; ``None`` clears. Bit ``b`` of ``local_mask``: the force on
        body ``b`` is expressed in the body frame (``pybullet_backend.py:603-658``)."""
        if force is not None:
            self._check_tensor(force, (self.n, _abi.NB, 3), name="force")
        check(lib().upkie_b200_set_external_forces(self._h, _ptr(force), int(local_mask), self._stream()))
        torch.cuda.current_stream(self.device).synchronize()
        self._external = (None if force is None else force.clone(), int(local_mask))

    def reset(
        self,
        mask: Optional[torch.Tensor] = None,
        init_state: Optional[torch.Tensor] = None,
        seed: int = 0,
        env_offset: int = 0,
    ) -> None:
        """``PyBulletBackend.reset`` for the envs selected by ``mask`` (all if
        None). ``init_state[N, 25]`` = sampled ``RobotState`` rows; None = sample
        on the device."""
        if mask is not None:
            self._check_tensor(mask, (self.n,), torch.uint8, "mask")
        if init_state is not None:
            self._check_tensor(init_state, (self.n, _abi.INIT_DIM), name="init_state")
        check(lib().upkie_b200_reset(self._h, _ptr(mask), _ptr(init_state), int(seed), int(env_offset), self._stream()))

    def _outputs(self, obs, default_obs, reward, terminated, truncated):
        """Caller-provided output tensors (e.g. ``RolloutBuffer.slot(t)``: the kernel then
        writes the rollout in place) or the handle's own."""
        obs = default_obs if obs is None else obs
        reward = self.reward if reward is None else reward
        terminated = self.terminated if terminated is None else terminated
        truncated = self.truncated if truncated is None else truncated
        if obs is not default_obs:
            if obs.numel() != default_obs.numel() or obs.data_ptr() % 16 != 0:
                raise UpkieRuntimeError("obs: wrong number of elements or not 16-byte aligned")
            self._check_tensor(obs, obs.shape, name="obs")
        if reward is not self.reward:
            self._check_tensor(reward, (self.n,), name="reward")
        if terminated is not self.terminated:
            self._check_tensor(terminated, (self.n,), torch.uint8, "terminated")
        if truncated is not self.truncated:
            self._check_tensor(truncated, (self.n,), torch.uint8, "truncated")
        return obs, reward, terminated, truncated

    def _step(self, act_dim: int, action, obs, reward, terminated, truncated, final_obs, compact: bool = False,
              final_state: bool = False):
        """``upkie_b200_step``: the general device-buffer step (``truncated`` with compact rows, ``final_obs``,
        ``final_state``)."""
        out = _abi.UpkieStepOutputs(_addr(obs), _addr(reward), _addr(terminated), _addr(truncated), _addr(final_obs),
                                    1 if compact else 0, 1 if final_state else 0)
        check(lib().upkie_b200_step(self._h, int(act_dim), _ptr(action), C.byref(out), self._stream()))

    def _check_final_obs(self, final_obs: Optional[torch.Tensor], shape):
        if final_obs is not None:
            self._check_tensor(final_obs, shape, name="final_obs")

    def step_servos(self, action: torch.Tensor, obs: Optional[torch.Tensor] = None, reward=None, terminated=None,
                    truncated=None, final_obs: Optional[torch.Tensor] = None, final_state: bool = False):
        """``final_obs[N, 6, 5]`` (same-step auto-reset): the envs that reset in this step first store there the
        observation they reached; the other rows are left untouched (mask with ``terminated | truncated``).
        ``final_state=True`` (same-step auto-reset): they also stash their pre-reset state, whose spine observation
        ``final_spine_obs()`` returns until the simulator moves on."""
        self._check_tensor(action, (self.n, 6, 6), name="action")
        obs, reward, terminated, truncated = self._outputs(obs, self.obs_servos, reward, terminated, truncated)
        if final_obs is not None or final_state:
            self._check_final_obs(final_obs, (self.n, 6, 5))
            self._step(36, action, obs, reward, terminated, truncated, final_obs, final_state=final_state)
            return obs, reward, terminated, truncated
        check(
            lib().upkie_b200_step_servos(
                self._h, _ptr(action), _ptr(obs), _ptr(reward), _ptr(terminated), _ptr(truncated), self._stream(),
            )
        )
        return obs, reward, terminated, truncated

    def step_servos_compact(self, action: torch.Tensor, obs: Optional[torch.Tensor] = None, terminated=None):
        """Device buffers, compact rows: ``obs[N, 6, 3]`` (position, velocity, torque) and ``terminated``; the
        constants of the reference (temperature, voltage, reward, truncated) are not written. What a rollout
        buffer gathered across GPUs carries (``RolloutBuffer(..., compact=True)``)."""
        self._check_tensor(action, (self.n, 6, 6), name="action")
        if obs is None:
            if getattr(self, "obs_servos_compact", None) is None:
                self.obs_servos_compact = torch.empty((self.n, 6, 3), dtype=torch.float32, device=self.device)
            obs = self.obs_servos_compact
        elif obs.numel() != self.n * 18 or obs.dtype != torch.float32 or not obs.is_contiguous() or obs.data_ptr() % 16:
            raise UpkieRuntimeError("obs: expected contiguous 16-byte aligned float32 [N, 6, 3]")
        terminated = self.terminated if terminated is None else terminated
        if terminated is not self.terminated:
            self._check_tensor(terminated, (self.n,), torch.uint8, "terminated")
        check(lib().upkie_b200_step_servos_compact(self._h, _ptr(action), _ptr(obs), _ptr(terminated), self._stream()))
        return obs, terminated

    def step_servos_compact_truncated(self, action: torch.Tensor, obs: Optional[torch.Tensor] = None, terminated=None,
                                      truncated=None, final_obs: Optional[torch.Tensor] = None,
                                      final_state: bool = False):
        """``step_servos_compact`` that also returns ``truncated`` (the episode time limit, ``max_episode_steps``)
        and, in same-step auto-reset mode, fills the compact rows ``final_obs[N, 6, 3]`` of the envs that reset.
        Returns ``(obs, terminated, truncated)``."""
        self._check_tensor(action, (self.n, 6, 6), name="action")
        if obs is None:
            if getattr(self, "obs_servos_compact", None) is None:
                self.obs_servos_compact = torch.empty((self.n, 6, 3), dtype=torch.float32, device=self.device)
            obs = self.obs_servos_compact
        elif obs.numel() != self.n * 18 or obs.dtype != torch.float32 or not obs.is_contiguous() or obs.data_ptr() % 16:
            raise UpkieRuntimeError("obs: expected contiguous 16-byte aligned float32 [N, 6, 3]")
        terminated = self.terminated if terminated is None else terminated
        truncated = self.truncated if truncated is None else truncated
        for name, t in (("terminated", terminated), ("truncated", truncated)):
            self._check_tensor(t, (self.n,), torch.uint8, name)
        self._check_final_obs(final_obs, (self.n, 6, 3))
        self._step(36, action, obs, None, terminated, truncated, final_obs, compact=True, final_state=final_state)
        return obs, terminated, truncated

    def step_servos_multicast(self, action: torch.Tensor, obs_mc_ptr: int, terminated_mc_ptr: int) -> None:
        """Compact rows and ``terminated`` go to NVSwitch multicast addresses (``PeerRolloutBuffer.multicast_slot``): every GPU of the node receives them."""
        self._check_tensor(action, (self.n, 6, 6), name="action")
        check(lib().upkie_b200_step_servos_multicast(
            self._h, _ptr(action), C.c_void_p(int(obs_mc_ptr)), C.c_void_p(int(terminated_mc_ptr)), self._stream()))

    def step_servos_peers(self, action: torch.Tensor, obs_ptrs, terminated_ptrs) -> None:
        """Compact rows and ``terminated`` stored by the step kernel into every buffer of ``obs_ptrs`` /
        ``terminated_ptrs`` (device addresses of this step's slot in each peer's symmetric rollout buffer,
        ``PeerRolloutBuffer.peer_slots``): the rollout gather over plain NVLink stores, no collective kernel."""
        self._check_tensor(action, (self.n, 6, 6), name="action")
        k = len(obs_ptrs)
        oa = (C.c_void_p * k)(*[C.c_void_p(int(x)) for x in obs_ptrs])
        ta = (C.c_void_p * k)(*[C.c_void_p(int(x)) for x in terminated_ptrs])
        check(lib().upkie_b200_step_servos_peers(self._h, _ptr(action), oa, ta, k, self._stream()))

    def step_servos_push(self, action: torch.Tensor, obs_ptr: int, terminated_ptr: int, push=None) -> None:
        """Deferred rollout transport (``upkie_b200_step_servos_push``): this step's compact rows go to the local slot
        at ``obs_ptr`` / ``terminated_ptr``; ``push`` (an ``_abi.UpkiePush`` from ``PeerRolloutBuffer.push_descriptor``)
        names an earlier slot the same launch sends to every GPU in its prologue, or None."""
        self._check_tensor(action, (self.n, 6, 6), name="action")
        check(lib().upkie_b200_step_servos_push(
            self._h, _ptr(action), C.c_void_p(int(obs_ptr)), C.c_void_p(int(terminated_ptr)),
            C.byref(push) if push is not None else None, self._stream()))

    def push_rows(self, push) -> None:
        """Send one slot on its own (last step of a rollout): ``upkie_b200_push_rows``."""
        check(lib().upkie_b200_push_rows(self._h, C.byref(push), self._stream()))

    def step_gyropod(self, action: torch.Tensor, obs: Optional[torch.Tensor] = None, reward=None, terminated=None,
                     truncated=None, final_obs: Optional[torch.Tensor] = None, final_state: bool = False):
        self._check_tensor(action, (self.n, 2), name="action")
        obs, reward, terminated, truncated = self._outputs(obs, self.obs_gyropod, reward, terminated, truncated)
        if final_obs is not None or final_state:
            self._check_final_obs(final_obs, (self.n, 6))
            self._step(2, action, obs, reward, terminated, truncated, final_obs, final_state=final_state)
            return obs, reward, terminated, truncated
        check(
            lib().upkie_b200_step_gyropod(
                self._h, _ptr(action), 2, _ptr(obs), _ptr(reward), _ptr(terminated), _ptr(truncated), self._stream(),
            )
        )
        return obs, reward, terminated, truncated

    def step_pendulum(self, action: torch.Tensor, obs: Optional[torch.Tensor] = None, reward=None, terminated=None,
                      truncated=None, final_obs: Optional[torch.Tensor] = None, final_state: bool = False):
        self._check_tensor(action, (self.n, 1), name="action")
        obs, reward, terminated, truncated = self._outputs(obs, self.obs_pendulum, reward, terminated, truncated)
        if final_obs is not None or final_state:
            self._check_final_obs(final_obs, (self.n, 4))
            self._step(1, action, obs, reward, terminated, truncated, final_obs, final_state=final_state)
            return obs, reward, terminated, truncated
        check(
            lib().upkie_b200_step_gyropod(
                self._h, _ptr(action), 1, _ptr(obs), _ptr(reward), _ptr(terminated), _ptr(truncated), self._stream(),
            )
        )
        return obs, reward, terminated, truncated

    # host-buffer path (H2D + kernel + D2H inside the call) ---------------------
    def _host_buffers(self):
        """Pinned host arrays owned by the handle: ``host_action_buffer()`` (fill it
        in place for a staging-free H2D copy) and the outputs returned by the
        ``*_host`` calls (overwritten by the next call)."""
        if getattr(self, "_hb", None) is None:
            def pinned(shape, dtype):
                return torch.empty(shape, dtype=dtype, pin_memory=True).numpy()

            self._hb = {
                "act36": pinned((self.n, 6, 6), torch.float32),
                "act2": pinned((self.n, 2), torch.float32),
                "act1": pinned((self.n, 1), torch.float32),
                "obs30": pinned((self.n, 6, 5), torch.float32),
                "obs18": pinned((self.n, 6, 3), torch.float32),
                "obs6": pinned((self.n, 6), torch.float32),
                "obs4": pinned((self.n, 4), torch.float32),
                "rew": pinned((self.n,), torch.float32),
                "term": pinned((self.n,), torch.uint8),
                "trunc": pinned((self.n,), torch.uint8),
                "trunc_dev": pinned((self.n,), torch.uint8),  # truncated as the kernel writes it (time limit set)
            }
            self._hb["rew"][:] = 0.0  # upkie_env.py:230
            self._hb["trunc"][:] = 0  # upkie_env.py:197
        return self._hb

    def _limited(self) -> bool:
        return self.config.max_episode_steps > 0

    def _host_final_obs(self, dim: int) -> np.ndarray:
        """Pinned final-observation rows of the same-step auto-reset (allocated on first use)."""
        hb = self._host_buffers()
        key = f"fin{dim}"
        if key not in hb:
            shape = {30: (self.n, 6, 5), 18: (self.n, 6, 3)}.get(dim, (self.n, dim))
            hb[key] = torch.zeros(shape, dtype=torch.float32, pin_memory=True).numpy()
        return hb[key]

    def host_action_buffer(self, act_dim: int = 36) -> np.ndarray:
        """Pinned ``[N, 6, 6]`` / ``[N, 2]`` / ``[N, 1]`` action array to fill in place."""
        return self._host_buffers()[f"act{act_dim}"]

    def step_servos_host(self, action: np.ndarray):
        """``action[N, 6, 6]`` float32 on the host (ideally ``host_action_buffer()``).
        Returns pinned arrays that the next ``*_host`` call overwrites."""
        hb = self._host_buffers()
        a = action
        if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
            a = np.ascontiguousarray(action, dtype=np.float32)
        if a.size != self.n * 36:
            raise UpkieRuntimeError(f"action: expected {self.n * 36} float32 values, got {a.size}")
        obs, rew, term = hb["obs30"], hb["rew"], hb["term"]
        # reward is a constant of the reference (upkie_env.py:230), and so is truncated without a time limit
        # (upkie_env.py:197): not transported then
        trunc = hb["trunc_dev"] if self._limited() else hb["trunc"]
        check(lib().upkie_b200_step_servos_host(self._h, a.ctypes.data, obs.ctypes.data, None, term.ctypes.data,
                                                trunc.ctypes.data if self._limited() else None))
        return obs, rew, term, trunc

    def step_servos_host_compact(self, action: np.ndarray):
        """Like ``step_servos_host`` but only the changing part of the observation crosses PCIe:
        returns ``obs[N, 6, 3]`` (position, velocity, torque per joint) and ``terminated``; temperature,
        voltage, reward and truncated are constants of the reference the caller fills once."""
        hb = self._host_buffers()
        a = action
        if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
            a = np.ascontiguousarray(action, dtype=np.float32)
        if a.size != self.n * 36:
            raise UpkieRuntimeError(f"action: expected {self.n * 36} float32 values, got {a.size}")
        obs, term = hb["obs18"], hb["term"]
        check(lib().upkie_b200_step_servos_host_compact(self._h, a.ctypes.data, obs.ctypes.data, term.ctypes.data))
        return obs, term

    def step_gyropod_host(self, action: np.ndarray):
        hb = self._host_buffers()
        a = np.ascontiguousarray(action, dtype=np.float32)
        act_dim = a.shape[1] if a.ndim == 2 else a.size // self.n
        if act_dim not in (1, 2) or a.size != self.n * act_dim:
            raise UpkieRuntimeError("action: expected shape [N, 1] (pendulum) or [N, 2] (gyropod)")
        obs = hb["obs6"] if act_dim == 2 else hb["obs4"]
        rew, term = hb["rew"], hb["term"]
        trunc = hb["trunc_dev"] if self._limited() else hb["trunc"]
        check(
            lib().upkie_b200_step_gyropod_host(self._h, a.ctypes.data, act_dim, obs.ctypes.data, None, term.ctypes.data,
                                               trunc.ctypes.data if self._limited() else None)
        )
        return obs, rew, term, trunc

    def step_host(self, action: np.ndarray, act_dim: int, compact: bool = False, final_obs: bool = False,
                  final_state: bool = False):
        """``upkie_b200_step_host``: host arrays, ``truncated`` written by the kernel on every path. ``act_dim`` 36
        (servos, ``compact`` = rows ``[N, 6, 3]``), 2 (gyropod) or 1 (pendulum). ``final_obs=True`` (same-step
        auto-reset): the envs that reset in this step also store the observation they reached into a pinned buffer
        of the observation's layout; its other rows keep their values. ``final_state=True``: they stash their
        pre-reset state in device memory (``final_spine_obs()``). Returns ``(obs, terminated, truncated, final_obs or
        None)``: pinned arrays that the next ``*_host`` call overwrites."""
        hb = self._host_buffers()
        a = action
        if a.dtype != np.float32 or not a.flags["C_CONTIGUOUS"]:
            a = np.ascontiguousarray(action, dtype=np.float32)
        if act_dim not in (36, 2, 1) or a.size != self.n * act_dim or (compact and act_dim != 36):
            raise UpkieRuntimeError(f"action: expected {self.n} rows of {act_dim} float32 values (act_dim 36, 2 or 1)")
        dim = {36: 18 if compact else 30, 2: 6, 1: 4}[act_dim]
        obs, term, trunc = hb[f"obs{dim}"], hb["term"], hb["trunc_dev"]
        fin = self._host_final_obs(dim) if final_obs else None
        out = _abi.UpkieStepOutputs(_addr(obs), None, _addr(term), _addr(trunc), _addr(fin), 1 if compact else 0,
                                    1 if final_state else 0)
        check(lib().upkie_b200_step_host(self._h, int(act_dim), a.ctypes.data, C.byref(out)))
        return obs, term, trunc, fin

    @property
    def launches(self) -> int:
        """Step kernels launched through this handle, counted by the library (bench.py's ``gpu_launches``)."""
        c = C.c_uint64(0)
        check(lib().upkie_b200_launch_count(self._h, C.byref(c)))
        return int(c.value)

    # ------------------------------------------------------------------
    def spine_obs(self) -> torch.Tensor:
        """``get_spine_observation`` for all envs, flattened ``[N, 62]``."""
        out = torch.empty((self.n, _abi.SPINE_DIM), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_spine_obs(self._h, _ptr(out), self._stream()))
        return out

    def final_spine_obs(self, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """Spine observations ``[N, 62]`` of the terminal step of the same-step auto-resets of the last step, which
        must have been taken with ``final_state=True`` (Gymnasium's ``info["final_info"]``): row ``i`` of an env that
        reset is what ``spine_obs()`` would have returned after that step without the reset. The other rows of
        ``out`` (zeros when ``out`` is None) are left untouched. Raises once the simulator has been stepped or reset
        again."""
        if out is None:
            out = torch.zeros((self.n, _abi.SPINE_DIM), dtype=torch.float32, device=self.device)
        else:
            self._check_tensor(out, (self.n, _abi.SPINE_DIM), name="out")
        check(lib().upkie_b200_final_spine_obs(self._h, _ptr(out), self._stream()))
        return out

    def reset_obs(self, obs_dim: int) -> torch.Tensor:
        shape = (self.n, 6, 5) if obs_dim == 30 else (self.n, obs_dim)
        out = torch.empty(shape, dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_reset_obs(self._h, int(obs_dim), _ptr(out), self._stream()))
        return out

    def get_state(self) -> torch.Tensor:
        out = torch.empty((self.n, _abi.STATE_DIM), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_state(self._h, _ptr(out), self._stream()))
        return out

    def get_body_contacts(self) -> torch.Tensor:
        """Body-ground contacts of the last substep, ``[n, BODY_REC_DIM]``: bit mask of the model's collision points that
        held contact rows, then per slot (collision point index, normal impulse, friction impulses along world -y and
        +x). What ``PyBulletBackend.get_contact_points`` reports for links other than the tires
        (``pybullet_backend.py:660-716``)."""
        out = torch.empty((self.n, _abi.BODY_REC_DIM), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_body_contacts(self._h, _ptr(out), self._stream()))
        return out

    def get_lag(self) -> torch.Tensor:
        """Spine mode: the lag records ``[N, LAG_DIM]`` (servo replies of the last two cycles, last IMU reading, the
        last assembled observation; ``include/upkie_b200.h`` ``UPKIE_LAG_*``)."""
        out = torch.empty((self.n, _abi.LAG_DIM), dtype=torch.float32, device=self.device)
        check(lib().upkie_b200_get_lag(self._h, _ptr(out), self._stream()))
        return out

    def set_lag(self, lag: torch.Tensor) -> None:
        self._check_tensor(lag, (self.n, _abi.LAG_DIM), name="lag")
        check(lib().upkie_b200_set_lag(self._h, _ptr(lag), self._stream()))

    def set_state(self, state: torch.Tensor) -> None:
        self._check_tensor(state, (self.n, _abi.STATE_DIM), name="state")
        check(lib().upkie_b200_set_state(self._h, _ptr(state), self._stream()))

    # checkpoint / resume ------------------------------------------------------------------
    def state_dict(self) -> dict:
        """Everything a handle needs to continue bit for bit (``torch.save``-able): robot state, episode / tick
        counters, time-limit counts, pending auto-resets, error flags, randomisation, per-env parameter table, external forces, auto-reset keys. The model and
        the configuration are construction arguments and are not included."""
        i32, u8 = torch.int32, torch.uint8
        episode = torch.empty(self.n, dtype=i32, device=self.device)
        tick = torch.empty(self.n, dtype=i32, device=self.device)
        pending = torch.empty(self.n, dtype=u8, device=self.device)
        flags = torch.empty(self.n, dtype=i32, device=self.device)
        check(lib().upkie_b200_get_counters(self._h, _ptr(episode), _ptr(tick), _ptr(pending), _ptr(flags), self._stream()))
        elapsed = torch.empty(self.n, dtype=i32, device=self.device)
        check(lib().upkie_b200_get_elapsed(self._h, _ptr(elapsed), self._stream()))
        friction, eps = getattr(self, "_randomization", (None, None))
        env_params = getattr(self, "_env_params", None)
        if getattr(self, "_randomized_at_reset", False):
            # resets drew on the device: the values in force are the device's
            friction, eps = self.get_randomization()
            env_params = self.get_env_params()
        spec = getattr(self, "_reset_randomization", None)
        push = getattr(self, "_push_randomization", None)
        push_count, push_timer = self.get_push_state()
        delay_count, delay_delay, delay_command = self.get_action_delay_state()
        sense_count, sense_delay, sense_rows = self.get_observation_delay_state()
        force, local_mask = getattr(self, "_external", (None, 0))
        sd = {
            "reset_randomization": None if spec is None else bytes(spec),  # the UpkieResetRandomization in force
            "draws": self.get_draws(),  # per-env draw counters of the reset randomisation
            "push_randomization": None if push is None else bytes(push),  # the UpkiePushRandomization in force
            "push_count": push_count, "push_timer": push_timer,  # per-env push schedule state
            "action_delay": getattr(self, "_action_delay", None),  # (substeps_low, substeps_high) in force, or None
            # per-env action-delay state: draw counters, delays, previous servo commands
            "action_delay_count": delay_count, "action_delay_delay": delay_delay,
            "action_delay_command": delay_command,
            # (substeps_low, substeps_high) of the observation delay in force, or None
            "observation_delay": getattr(self, "_observation_delay", None),
            # per-env observation-delay state: draw counters, delays, sensed state rows
            "observation_delay_count": sense_count, "observation_delay_delay": sense_delay,
            "observation_delay_rows": sense_rows,
        }
        # delays of more than one tick: the depth and the history of each (absent at depth 1, as before the histories
        # existed), also while the delay is off: the handle keeps its history for a later spec of the same depth
        delay_ticks = getattr(self, "_action_delay_ticks", 1)
        if delay_ticks > 1:
            sd["action_delay_ticks"] = delay_ticks
            sd["action_delay_history"] = self.get_action_delay_history()
        sense_ticks = getattr(self, "_observation_delay_ticks", 1)
        if sense_ticks > 1:
            sd["observation_delay_ticks"] = sense_ticks
            sd["observation_delay_history"] = self.get_observation_delay_history()
        # the observation history: (columns, size) and its ring in age order (absent without one)
        if self.history_spec is not None:
            sd["history"] = self.history_spec
            sd["history_ring"] = self.get_history_state()
        # the servo dropouts: (prob_low, prob_high, joint_mask) and the per-env state (absent without a spec)
        if self.servo_dropout_spec is not None:
            sd["servo_dropout"] = self.servo_dropout_spec
            sd["servo_dropout_count"], sd["servo_dropout_prob"], sd["servo_dropout_held"] = \
                self.get_servo_dropout_state()
        # the IMU misalignment: its ranges and the per-env state (absent without a spec)
        if self.imu_misalignment_spec is not None:
            sd["imu_misalignment"] = self.imu_misalignment_spec
            sd["imu_misalignment_count"], sd["imu_misalignment_quat"] = self.get_imu_misalignment_state()
        # the encoder offsets: (low, high, joint_mask) and the per-env state (absent without a spec)
        if self.encoder_offset_spec is not None:
            sd["encoder_offset"] = self.encoder_offset_spec
            sd["encoder_offset_count"], sd["encoder_offset_offset"] = self.get_encoder_offset_state()
        # the servo noise: its ranges and the per-env state (absent without a spec)
        if self.servo_noise_spec is not None:
            sd["servo_noise"] = self.servo_noise_spec
            sd["servo_noise_count"], sd["servo_noise_sigma"] = self.get_servo_noise_state()
            sd["servo_noise_mark"] = self.get_servo_noise_mark()
        # the velocity limits: (max_velocity, derate, joint_mask) and the per-env state (absent without a spec)
        if self.velocity_derate_spec is not None:
            sd["velocity_derate"] = self.velocity_derate_spec
            sd["velocity_derate_count"], sd["velocity_derate_max_velocity"] = self.get_velocity_derate_state()
        # the torque scales: (scale, joint_mask) and the per-env state (absent without a spec)
        if self.torque_scale_spec is not None:
            sd["torque_scale"] = self.torque_scale_spec
            sd["torque_scale_count"], sd["torque_scale_scale"] = self.get_torque_scale_state()
        # the attitude filter: its ranges and the per-env state (absent without a spec)
        if self.attitude_filter_spec is not None:
            sd["attitude_filter"] = self.attitude_filter_spec
            (sd["attitude_filter_count"], sd["attitude_filter_gains"], sd["attitude_filter_quat"],
             sd["attitude_filter_bias"]) = self.get_attitude_filter_state()
            sd["attitude_filter_report"] = self.get_attitude_filter_report()
        sd.update({
            "lag": self.get_lag() if self.config.spine_mode else None,  # spine mode: replies / IMU of the last cycles
            "state": self.get_state(), "episode": episode, "tick": tick, "pending_reset": pending, "error_flags": flags,
            "elapsed": elapsed,  # steps since each env's last reset (the time limit's counts)
            "friction": friction, "inertia_eps": eps, "external_force": force, "external_local_mask": local_mask,
            "env_params": env_params,  # per-env parameter table, None = the config's values
            "autoreset": getattr(self, "_autoreset", (AUTORESET_DISABLED, 0, 0)),
        })
        return sd

    def load_state_dict(self, sd: dict) -> None:
        dev = self.device
        # the attitude filter is off while the state and the observation delay are restored (set_state re-initialises
        # its estimates, and a handle with a filter refuses a delay of more than one tick), and restored last
        self.set_attitude_filter(None)
        self.set_state(sd["state"].to(dev))
        if sd.get("lag") is not None:
            self.set_lag(sd["lag"].to(dev))
        check(lib().upkie_b200_set_counters(
            self._h, _ptr(sd["episode"].to(dev)), _ptr(sd["tick"].to(dev)), _ptr(sd["pending_reset"].to(dev)),
            _ptr(sd["error_flags"].to(dev)), self._stream()))
        # a checkpoint written before the time limit existed restores zero counts
        elapsed = sd.get("elapsed")
        elapsed = torch.zeros(self.n, dtype=torch.int32, device=dev) if elapsed is None else elapsed.to(dev).contiguous()
        check(lib().upkie_b200_set_elapsed(self._h, _ptr(elapsed), self._stream()))
        torch.cuda.current_stream(dev).synchronize()
        # the servo noise is off while the observation delay and the servo dropouts are restored (a handle with noise
        # refuses the second of the two), and restored last
        self.set_servo_noise(None)
        # the buffers a reset randomisation spec writes into are restored with the spec off; a checkpoint written
        # before reset randomisation existed loads as "off, counters 0"
        if getattr(self, "_reset_randomization", None) is not None:
            self.set_reset_randomization(None)
        # so is the push spec (it would refuse a checkpoint's body-frame force on its body); a checkpoint written before
        # push randomisation existed loads as "off, counters 0"
        self.set_push_randomization(None)
        self.set_randomization(None if sd["friction"] is None else sd["friction"].to(dev),
                               None if sd["inertia_eps"] is None else sd["inertia_eps"].to(dev))
        self.set_external_forces(None if sd["external_force"] is None else sd["external_force"].to(dev),
                                 sd["external_local_mask"])
        # a checkpoint written before the per-env parameter table existed loads as "no table"
        env_params = sd.get("env_params")
        self.set_env_params(None if env_params is None else env_params.to(dev).contiguous())
        spec = sd.get("reset_randomization")
        if spec is not None:
            self.set_reset_randomization(_abi.UpkieResetRandomization.from_buffer_copy(spec))
        draws = sd.get("draws")
        if spec is not None or getattr(self, "_randomized_at_reset", False) or (draws is not None and bool(draws.any())):
            draws = torch.zeros(self.n, dtype=torch.int32, device=dev) if draws is None else draws.to(dev).contiguous()
            self.set_draws(draws)
        push = sd.get("push_randomization")
        if push is not None:
            self.set_push_randomization(_abi.UpkiePushRandomization.from_buffer_copy(push))
        zeros = torch.zeros(self.n, dtype=torch.int32, device=dev)
        count, timer = sd.get("push_count"), sd.get("push_timer")
        self.set_push_state(zeros if count is None else count.to(dev).contiguous(),
                            zeros if timer is None else timer.to(dev).contiguous())
        # a checkpoint written before the action delay existed loads as "off, counters 0, delays 0" (and stop rows)
        delay = sd.get("action_delay")
        delay_ticks = int(sd.get("action_delay_ticks", 1))  # a checkpoint without a history is depth 1
        if delay is None:
            if delay_ticks != getattr(self, "_action_delay_ticks", 1):  # the depth of a delay that is off: set with a spec that draws nothing, then off
                self.set_action_delay(0, 0, max_ticks=delay_ticks)
            self.set_action_delay(None)
        else:
            self.set_action_delay(*delay, max_ticks=delay_ticks)
        count, delay_d, command = (sd.get(k) for k in ("action_delay_count", "action_delay_delay",
                                                       "action_delay_command"))
        stop = stop_commands(self.n, dev)
        default = count is None or (not count.any() and not delay_d.any()
                                    and torch.equal(command.to(dev).nan_to_num(7.0), stop.nan_to_num(7.0)))
        if delay is not None or not default or getattr(self, "_delay_state_set", False):
            # the handle's state is replaced; a handle that never had one and a checkpoint without one (no spec and
            # the state of a fresh handle) leave the buffers unallocated
            self.set_action_delay_state(zeros if count is None else count.to(dev).contiguous(),
                                        zeros if delay_d is None else delay_d.to(dev).contiguous(),
                                        stop if command is None else command.to(dev).contiguous())
        if sd.get("action_delay_history") is not None:
            self.set_action_delay_history(sd["action_delay_history"].to(dev).contiguous())
        # a checkpoint written before the observation delay existed loads as "off, counters 0, delays 0" (and the
        # state as the sensed rows)
        sense = sd.get("observation_delay")
        sense_ticks = int(sd.get("observation_delay_ticks", 1))
        if sense is None:
            if sense_ticks != getattr(self, "_observation_delay_ticks", 1):  # as the action delay's (the state and the history are restored below)
                self.set_observation_delay(0, 0, max_ticks=sense_ticks)
            self.set_observation_delay(None)
        else:
            self.set_observation_delay(*sense, max_ticks=sense_ticks)
        count, delay_d, rows = (sd.get(k) for k in ("observation_delay_count", "observation_delay_delay",
                                                    "observation_delay_rows"))
        state = sd["state"].to(dev)
        default = count is None or (not count.any() and not delay_d.any()
                                    and torch.equal(rows.to(dev).nan_to_num(7.0), state.nan_to_num(7.0)))
        if sense is not None or not default or getattr(self, "_sense_state_set", False):
            # as the action delay's: a handle that never had a state and a checkpoint without one allocate nothing
            self.set_observation_delay_state(zeros if count is None else count.to(dev).contiguous(),
                                             zeros if delay_d is None else delay_d.to(dev).contiguous(),
                                             state.contiguous() if rows is None else rows.to(dev).contiguous())
        if sd.get("observation_delay_history") is not None:
            self.set_observation_delay_history(sd["observation_delay_history"].to(dev).contiguous())
        # the observation history after the observation delay, whose depth sizes its ring; a checkpoint without one
        # turns it off
        hist = sd.get("history")
        self.set_history(None if hist is None else hist[0], 1 if hist is None else hist[1])
        if hist is not None:
            self.set_history_state(sd["history_ring"].to(dev).contiguous())
        # the servo dropouts; a checkpoint without them (or written before they existed) turns them off
        drop = sd.get("servo_dropout")
        if drop is None:
            self.set_servo_dropout(None)
        else:
            self.set_servo_dropout(drop[0], drop[1], [n for j, n in enumerate(_abi.JOINT_NAMES) if (drop[2] >> j) & 1])
            self.set_servo_dropout_state(*(sd[k].to(dev).contiguous() for k in (
                "servo_dropout_count", "servo_dropout_prob", "servo_dropout_held")))
        # the IMU misalignment; a checkpoint without one (or written before it existed) turns it off
        tilt = sd.get("imu_misalignment")
        if tilt is None:
            self.set_imu_misalignment(None)
        else:
            self.set_imu_misalignment(*tilt)
            self.set_imu_misalignment_state(*(sd[k].to(dev).contiguous() for k in (
                "imu_misalignment_count", "imu_misalignment_quat")))
        # the encoder offsets; a checkpoint without them (or written before they existed) turns them off
        enc = sd.get("encoder_offset")
        if enc is None:
            self.set_encoder_offset(None)
        else:
            self.set_encoder_offset(enc[0], enc[1], [n for j, n in enumerate(_abi.JOINT_NAMES) if (enc[2] >> j) & 1])
            self.set_encoder_offset_state(*(sd[k].to(dev).contiguous() for k in (
                "encoder_offset_count", "encoder_offset_offset")))
        # the velocity limits; a checkpoint without them (or written before they existed) turns them off
        vlim = sd.get("velocity_derate")
        if vlim is None:
            self.set_velocity_derate(None)
        else:
            self.set_velocity_derate(vlim[0], vlim[1], [n for j, n in enumerate(_abi.JOINT_NAMES) if (vlim[2] >> j) & 1])
            self.set_velocity_derate_state(*(sd[k].to(dev).contiguous() for k in (
                "velocity_derate_count", "velocity_derate_max_velocity")))
        # the torque scales; a checkpoint without them (or written before they existed) turns them off
        tsc = sd.get("torque_scale")
        if tsc is None:
            self.set_torque_scale(None)
        else:
            self.set_torque_scale(tsc[0], [n for j, n in enumerate(_abi.JOINT_NAMES) if (tsc[1] >> j) & 1])
            self.set_torque_scale_state(*(sd[k].to(dev).contiguous() for k in ("torque_scale_count", "torque_scale_scale")))
        # the servo noise (off above); a checkpoint without it (or written before it existed) leaves it off
        noise = sd.get("servo_noise")
        if noise is not None:
            self.set_servo_noise(*noise)
            self.set_servo_noise_state(*(sd[k].to(dev).contiguous() for k in ("servo_noise_count", "servo_noise_sigma")))
            if sd.get("servo_noise_mark") is not None:
                self.set_servo_noise_mark(sd["servo_noise_mark"].to(dev).contiguous())
        # the attitude filter (off above), after the state; a checkpoint without it (or written before it existed)
        # leaves it off
        att = sd.get("attitude_filter")
        if att is not None:
            self.set_attitude_filter(*att)
            self.set_attitude_filter_state(*(sd[k].to(dev).contiguous() for k in (
                "attitude_filter_count", "attitude_filter_gains", "attitude_filter_quat", "attitude_filter_bias")))
            self.set_attitude_filter_report(sd["attitude_filter_report"].to(dev).contiguous())
        self.set_autoreset(*sd["autoreset"])

    def error_flags(self) -> torch.Tensor:
        out = torch.empty(self.n, dtype=torch.int32, device=self.device)
        check(lib().upkie_b200_error_flags(self._h, _ptr(out), self._stream()))
        return out


def stop_commands(n: int, device=None) -> torch.Tensor:
    """``[n, 6, 6]`` stop rows, the servo command an env holds after a reset under an action delay: per joint position
    NaN, every other key 0 (``include/upkie_b200.h``)."""
    out = torch.zeros((n, _abi.NJ, len(_abi.ACT_KEYS)), dtype=torch.float32, device=device)
    out[:, :, 0] = float("nan")
    return out


def neutral_action(model: Model, n: int, device=None) -> torch.Tensor:
    """``UpkieServos.get_neutral_action`` (``upkie_servos.py:255-262``) as a
    ``[N, 6, 6]`` tensor."""
    a = torch.zeros((n, 6, 6), dtype=torch.float32, device=device)
    a[:, :, 0] = float("nan")
    a[:, :, 3] = 1.0
    a[:, :, 4] = 1.0
    a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device=device)
    return a
