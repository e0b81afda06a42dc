# SPDX-License-Identifier: Apache-2.0
"""Single-robot ``Backend`` on the GPU kernels.

``B200Backend`` implements the reference's backend interface
(``upkie/envs/backends/backend.py:11-50``: ``reset(init_state) -> dict``,
``step(action: dict) -> dict``, ``get_spine_observation() -> dict``, ``close()``, plus
``PyBulletBackend``'s ``randomize_inertias``, ``set_external_forces`` and ``get_contact_points``)
with one env of the vectorised simulation, so that the reference's own
``UpkieServos`` / ``UpkieGyropod`` / ``UpkiePendulum`` / ``UpkieBaseVelocity``
run unmodified on top of it (``UpkieServos(backend=B200Backend(dt=1/200))``).
It is the N = 1 compatibility path; throughput comes from ``B200VectorEnv``.

Action dictionary contract of ``PyBulletBackend.step``
(``pybullet_backend.py:276-300``): ``action["servo"][joint]`` must hold
``position`` (may be NaN), ``velocity`` and ``maximum_torque``;
``feedforward_torque`` defaults to 0, ``kp_scale`` / ``kd_scale`` to 1; joints
absent from the dictionary receive no torque; unknown joints are ignored;
``step({})`` is legal.
"""

from typing import Dict, List, Optional

import numpy as np
import torch

from . import _abi
from .envs import make_config, spine_row_to_dict
from .model import Model, PointContact, contact_points_from_state, default_model
from .robot_state import RobotState
from .sim import UpkieSim

try:  # derive from the reference's ABC when the reference package is importable
    from upkie.envs.backends.backend import Backend as _Base  # type: ignore
except Exception:  # pragma: no cover - the reference is not installed in this image

    class _Base:  # minimal stand-in with the same abstract surface
        pass


class B200Backend(_Base):
    """Backend using the sm_90a simulation kernels (one robot)."""

    def __init__(
        self,
        dt: float,
        gui: bool = False,
        inertia_variation: float = 0.0,
        joint_properties: Optional[Dict[str, object]] = None,
        model: Optional[Model] = None,
        nb_substeps: Optional[int] = None,
        torque_control_kd: float = 1.0,
        torque_control_kp: float = 20.0,
        device: int = 0,
        joint_limits: bool = True,
        body_contacts: bool = True,
    ) -> None:
        # same keyword arguments as PyBulletBackend.__init__ (pybullet_backend.py:55-66); gui is ignored.
        # joint_limits (extension): Bullet's hip / knee limit constraints, on as in the multibody loadURDF builds;
        # body_contacts (extension): the links' collision shapes rest on the floor, as in Bullet
        self.__dt = dt
        self.__model = model if model is not None else default_model()
        self.torque_control_kd = torque_control_kd
        self.torque_control_kp = torque_control_kp
        self.inertia_variation = inertia_variation
        cfg = make_config(
            frequency=1.0 / dt, nb_substeps=nb_substeps, torque_control_kp=torque_control_kp,
            torque_control_kd=torque_control_kd, joint_properties=joint_properties, joint_limits=joint_limits,
            body_contacts=body_contacts,
        )
        cfg.skip_action_clamps = 1  # the env on top (UpkieServos.get_spine_action) clamps, as in the reference
        self._sim = UpkieSim(1, model=self.__model, config=cfg, device=device)
        self._action = torch.zeros((1, 6, 6), dtype=torch.float32, device=self._sim.device)
        self._last_torque = np.zeros(6)
        self.joystick = None
        if abs(inertia_variation) > 1e-10:
            self.randomize_inertias(inertia_variation)

    def close(self) -> None:
        self._sim.close()

    def randomize_inertias(self, inertia_variation: float) -> None:
        """``PyBulletBackend.randomize_inertias`` (``pybullet_backend.py:571-601``)."""
        eps = np.random.default_rng().uniform(-inertia_variation, inertia_variation, size=(1, 6)).astype(np.float32)
        self._sim.set_randomization(inertia_eps=torch.from_numpy(eps).to(self._sim.device))

    def set_external_forces(self, external_forces: dict) -> None:
        """``PyBulletBackend.set_external_forces`` (``pybullet_backend.py:603-625``): forces persist, link
        by link, until overwritten."""
        self._external_forces = dict(getattr(self, "_external_forces", {}))
        self._external_forces.update(external_forces)
        rows, mask = self._sim.model.external_force_rows(self._external_forces, 1)
        self._sim.set_external_forces(torch.from_numpy(rows).to(self._sim.device), mask)

    def get_contact_points(self, link_name: Optional[str] = None) -> List[PointContact]:
        """``PyBulletBackend.get_contact_points`` (``pybullet_backend.py:660-716``): the contacts of the robot, or
        of one link of it, as of the last simulation substep. The simulated contacts are the two tire-ground
        points, reported on ``left_wheel_tire`` / ``right_wheel_tire``, and the collision points of the other links
        that touch the ground (the torso box of a fallen robot; DESIGN.md section 3). ``force_in_world`` sums the
        normal and the two friction components of the last substep, as the reference does
        (``pybullet_backend.py:696-709``)."""
        row = self._sim.get_state()[0].cpu().numpy()
        rec = self._sim.get_body_contacts()[0].cpu().numpy()
        return contact_points_from_state(self._sim.model, row, self._sim.config, link_name, rec)

    def reset(self, init_state: RobotState) -> dict:
        row = torch.from_numpy(init_state.to_row().astype(np.float32)).reshape(1, _abi.INIT_DIM).to(self._sim.device)
        self._sim.reset(init_state=row)
        return self.get_spine_observation()

    def step(self, action: dict) -> dict:
        a = np.zeros((6, 6), dtype=np.float32)
        a[:, _abi.ACT_KEYS.index("position")] = np.nan
        absent = []
        servo_actions = action.get("servo", {}) if action else {}
        for j, name in enumerate(_abi.JOINT_NAMES):
            sa = servo_actions.get(name)
            if sa is None:
                absent.append(j)  # no torque: zero gains and zero maximum torque
                continue
            velocity = float(sa["velocity"])
            assert not np.isnan(velocity)  # pybullet_backend.py:519
            a[j] = [
                float(sa["position"]),
                velocity,
                float(sa.get("feedforward_torque", 0.0)),
                float(sa.get("kp_scale", 1.0)),
                float(sa.get("kd_scale", 1.0)),
                float(sa["maximum_torque"]),
            ]
        self._action.copy_(torch.from_numpy(a).reshape(1, 6, 6))
        self._sim.step_servos(self._action)
        obs = self.get_spine_observation()
        for j in absent:  # the reference keeps the last commanded torque of joints it did not command
            obs["servo"][_abi.JOINT_NAMES[j]]["torque"] = float(self._last_torque[j])
        for j, name in enumerate(_abi.JOINT_NAMES):
            self._last_torque[j] = obs["servo"][name]["torque"]
        return obs

    def get_spine_observation(self) -> dict:
        row = self._sim.spine_obs()[0].cpu().numpy()
        return spine_row_to_dict(row)
