# SPDX-License-Identifier: Apache-2.0
"""upkie_b200 -- H100-native vectorised Upkie simulation and balance control.

Drop-in for the reference's env-step hot path (``UpkieServos`` /
``UpkieGyropod`` / ``UpkiePendulum`` / ``UpkieBaseVelocity`` on the PyBullet
backend, and ``MPCBalancer``); see DESIGN.md and INTEGRATION.md. Importing the
package needs neither a GPU nor the compiled library; creating an env does.
"""

__version__ = "0.1.0"

from . import _abi  # noqa: F401
from .exceptions import (  # noqa: F401
    MissingOptionalDependency,
    ModelError,
    UpkieException,
    UpkieRuntimeError,
)
from .model import ExternalForce, JointProperties, Model, default_model  # noqa: F401
from .robot_state import RobotState, RobotStateRandomization  # noqa: F401

_ACTIONS = {"Servos": "servos", "Gyropod": "gyropod", "Pendulum": "pendulum", "BaseVelocity": "base_velocity"}
# ``<Robot>-B200-<Action>``, the reference's ``<Robot>-<Backend>-<Action>`` scheme (``upkie/envs/__init__.py:24-44``)
ENV_IDS = {f"{robot}-B200-{name}": env_type for robot in ("Upkie", "Cookie") for name, env_type in _ACTIONS.items()}


def get_cookie_model() -> Model:
    """The Cookie robot (right-wheeled) from the ``cookie_description`` package, as
    ``upkie/envs/entry_points.py:295-308`` loads it; the package is an optional dependency there as well."""
    try:
        import cookie_description
    except ImportError as e:
        raise MissingOptionalDependency(
            "cookie_description not found, install it via `pip install cookie_description` "
            "or pass model=Model.from_urdf(path)"
        ) from e
    return Model.from_urdf(cookie_description.URDF_PATH)


def make_vec(env_id: str, num_envs: int, **kwargs):
    """``gymnasium.make_vec``-style factory for the ids of ``register()``. ``Cookie-B200-*`` ids load the Cookie
    model unless a ``model=`` is given (``make_cookie_pybullet_servos``, ``entry_points.py:311-336``)."""
    from .envs import B200VectorEnv

    if env_id not in ENV_IDS:
        raise UpkieException(f"unknown environment id {env_id!r}; known ids: {sorted(ENV_IDS)}")
    if env_id.startswith("Cookie-") and kwargs.get("model") is None:
        kwargs["model"] = get_cookie_model()
    return B200VectorEnv(num_envs, ENV_IDS[env_id], **kwargs)


def register() -> None:
    """Register ``{Upkie,Cookie}-B200-{Servos,Gyropod,Pendulum,BaseVelocity}`` with Gymnasium,
    following the reference's ``Upkie-<Backend>-<Action>`` scheme
    (``upkie/envs/__init__.py:24-44``). Needs gymnasium."""
    try:
        import gymnasium as gym
    except ImportError as e:
        raise MissingOptionalDependency("gymnasium not found; use upkie_b200.make_vec(...) directly") from e
    for env_id, env_type in ENV_IDS.items():
        if env_id in gym.registry:
            continue

        def vector_entry_point(num_envs=1, _id=env_id, **kwargs):
            return make_vec(_id, num_envs, **kwargs)

        gym.register(id=env_id, vector_entry_point=vector_entry_point)
