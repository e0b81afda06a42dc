# SPDX-License-Identifier: Apache-2.0
"""``UpkieBaseVelocity`` glue (``upkie/envs/upkie_base_velocity.py:164-202``) as device-agnostic tensor code.

The env is an MPC balancer in front of the gyropod env plus dead reckoning. ``base_velocity_tick`` states the
reference's ordering with the three heavy pieces (MPC solve, gyropod step, spine observation) passed in as
callables; the CPU tests bind the oracle and pin it on golden runs of the reference's own class
(``tests/test_base_velocity_golden.py``). ``B200VectorEnv`` runs the same ordering on the GPU with its epilogue (dead
reckoning, observation, and the auto-resets' ``UpkieBaseVelocity.reset``) in one kernel, ``base_velocity_post``.
"""
import ctypes as C
from typing import Callable, Optional, Tuple

import torch

from . import _abi
from ._lib import check, lib


def mpc_inputs_from_spine(spine_obs: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor]:
    """``MPCBalancer.step`` observation unpacking (``mpc_balancer.py:253-258``): state
    ``[ground position, base pitch, ground velocity, base pitch rate]`` and the floor-contact flag from flat spine
    observation rows ``[N, 62]``."""
    A = _abi
    x0 = torch.stack(
        [
            spine_obs[:, A.SP_ODOM_POS],
            spine_obs[:, A.SP_PITCH],
            spine_obs[:, A.SP_ODOM_VEL],
            spine_obs[:, A.SP_BASE_ANGVEL + 1],
        ],
        dim=1,
    ).contiguous()
    contact = (spine_obs[:, A.SP_CONTACT] > 0.5).to(torch.uint8)
    return x0, contact


def base_velocity_tick(
    action: torch.Tensor,
    spine: torch.Tensor,
    xy: torch.Tensor,
    dt: float,
    mpc_step_spine: Callable[[torch.Tensor, torch.Tensor, float], torch.Tensor],
    step_gyropod: Callable[[torch.Tensor], Tuple[torch.Tensor, torch.Tensor, torch.Tensor, torch.Tensor]],
    spine_obs: Callable[[], torch.Tensor],
):
    """One ``UpkieBaseVelocity.step``: the MPC turns the commanded linear velocity ``action[:, 0]`` into a ground
    velocity from the LAST spine observation (the one the previous step or the reset returned), the gyropod env is
    stepped with ``[ground velocity, action[:, 1]]``, and ``xy`` (updated in place) dead-reckons the COMMANDED linear
    velocity along the POST-step yaw. Returns ``(obs[N, 3], reward, terminated, truncated, new_spine)``."""
    linear_velocity = action[:, 0].contiguous()
    ground_velocity = mpc_step_spine(linear_velocity, spine, dt)
    gyro_action = torch.stack([ground_velocity, action[:, 1]], dim=1).contiguous()
    obs6, rew, term, trunc = step_gyropod(gyro_action)
    new_spine = spine_obs()
    yaw = obs6[:, 2]
    xy[:, 0] += linear_velocity * torch.cos(yaw) * dt
    xy[:, 1] += linear_velocity * torch.sin(yaw) * dt
    obs = torch.cat([xy, yaw[:, None]], dim=1)
    return obs, rew, term, trunc, new_spine


def _addr(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def base_velocity_post(sim, mpc_balancer, action: torch.Tensor, gyro_obs: torch.Tensor, xy: torch.Tensor, dt: float,
                       obs: torch.Tensor, autoreset_mode: int, gyro_final_obs: Optional[torch.Tensor] = None,
                       final_obs: Optional[torch.Tensor] = None) -> None:
    """``upkie_b200_base_velocity_post`` (``k_base_velocity_post``): the end of ``base_velocity_tick`` in one launch,
    after ``sim``'s gyropod step and spine observation. Envs that did not reset in this tick dead-reckon ``xy`` (in
    place) with the commanded linear velocity ``action[:, 0]`` along the post-step yaw ``gyro_obs[:, 2]`` and return
    ``[x, y, yaw]`` in ``obs[N, 3]``, with the bits of ``base_velocity_tick``'s torch arithmetic. Envs that a fused
    auto-reset of this tick re-initialised get ``UpkieBaseVelocity.reset`` (``upkie_base_velocity.py:137-162``):
    ``x = y = 0``, observation ``[0, 0, 0]``, ``mpc_balancer.commanded_velocity`` 0 and no warm start; in same-step mode
    (``autoreset_mode`` 2) they first store the ``[x, y, yaw]`` they reached, with the pre-reset yaw
    ``gyro_final_obs[:, 2]``, into ``final_obs[N, 3]`` (other rows untouched)."""
    n = sim.n
    sim._check_tensor(action, (n, 2), name="action")
    sim._check_tensor(gyro_obs, (n, 6), name="gyro_obs")
    sim._check_tensor(xy, (n, 2), name="xy")
    sim._check_tensor(obs, (n, 3), name="obs")
    sim._check_tensor(mpc_balancer.commanded_velocity, (n,), name="commanded_velocity")
    if gyro_final_obs is not None:
        sim._check_tensor(gyro_final_obs, (n, 6), name="gyro_final_obs")
    if final_obs is not None:
        sim._check_tensor(final_obs, (n, 3), name="final_obs")
    args = _abi.UpkieBaseVelocityPost(
        _addr(action), _addr(gyro_obs), _addr(gyro_final_obs), _addr(xy), _addr(mpc_balancer.commanded_velocity),
        _addr(obs), _addr(final_obs), float(dt), int(autoreset_mode))
    check(lib().upkie_b200_base_velocity_post(sim._h, mpc_balancer._h, C.byref(args), sim._stream()))
