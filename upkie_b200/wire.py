# SPDX-License-Identifier: Apache-2.0
"""Wire format of the reference's agent <-> spine mailbox, for replaying GPU trajectories against a real spine
(or a spine log against the GPU simulator).

The reference exchanges msgpack dictionaries through a POSIX shared-memory mailbox laid out as
``[request: u32][size: u32][payload]`` in native byte order (``upkie/envs/backends/spine/spine_interface.py:108-169``,
``upkie/cpp/spine/AgentInterface.cpp:70-97``); payloads are packed with
``msgpack.Packer(default=serialize, use_bin_type=True)`` where ``serialize`` turns arrays into lists
(``upkie/envs/backends/spine/serialize.py:8-37``) and unpacked with ``msgpack.Unpacker(raw=False)``.
This module produces and consumes exactly those bytes; it does not open any shared memory.
"""
import sys
from enum import IntEnum
from typing import Tuple

import msgpack
import numpy as np

from . import _abi


class Request(IntEnum):
    """``upkie/envs/backends/spine/request.py``"""

    kNone = 0
    kAction = 1
    kStart = 2
    kStop = 3
    kError = 4


def serialize(obj):
    """``upkie/envs/backends/spine/serialize.py:8-37``"""
    if hasattr(obj, "tolist"):
        return obj.tolist()
    elif hasattr(obj, "np"):
        return obj.np.tolist()
    elif hasattr(obj, "serialize"):
        return obj.serialize()
    return obj


def pack_dict(dictionary: dict) -> bytes:
    return msgpack.Packer(default=serialize, use_bin_type=True).pack(dictionary)


def unpack_dict(data: bytes) -> dict:
    unpacker = msgpack.Unpacker(raw=False)
    unpacker.feed(data)
    out = list(unpacker)
    if len(out) != 1:
        raise ValueError(f"expected one msgpack dictionary, got {len(out)}")
    return out[0]


def frame(request: int, payload: bytes = b"") -> bytes:
    """Mailbox image ``[request][size][payload]`` (``spine_interface.py:153-169``)."""
    return int(request).to_bytes(4, sys.byteorder) + len(payload).to_bytes(4, sys.byteorder) + payload


def parse_frame(buf: bytes) -> Tuple[Request, bytes]:
    request = Request(int.from_bytes(buf[0:4], sys.byteorder))
    size = int.from_bytes(buf[4:8], sys.byteorder)
    return request, bytes(buf[8:8 + size])


def action_row_to_dict(action: np.ndarray) -> dict:
    """One ``[6, 6]`` servo action (``ACTION_KEYS`` order) -> the spine action dictionary
    ``{"servo": {joint: {key: float}}}`` (``upkie_servos.py:308-344``)."""
    a = np.asarray(action, dtype=np.float64).reshape(6, 6)
    return {"servo": {name: {key: float(a[j, k]) for k, key in enumerate(_abi.ACT_KEYS)}
                      for j, name in enumerate(_abi.JOINT_NAMES)}}


def action_dict_to_row(action: dict) -> np.ndarray:
    """Spine action dictionary -> ``[6, 6]`` float32 with the backend's defaults for missing keys
    (``feedforward_torque = 0``, ``kp_scale = kd_scale = 1``, ``pybullet_backend.py:284-291``); joints absent
    from the dictionary get no torque (zero gains, zero maximum torque), unknown joints are ignored (``:280``)."""
    out = np.zeros((6, 6), dtype=np.float32)
    out[:, 0] = np.nan
    servo = (action or {}).get("servo", {})
    for j, name in enumerate(_abi.JOINT_NAMES):
        sa = servo.get(name)
        if sa is None:
            continue
        out[j] = [sa["position"], sa["velocity"], sa.get("feedforward_torque", 0.0), sa.get("kp_scale", 1.0),
                  sa.get("kd_scale", 1.0), sa["maximum_torque"]]
    return out


def pack_observation(spine_row: np.ndarray) -> bytes:
    """Flat spine observation row ``[62]`` -> the msgpack bytes a spine would have written."""
    from .envs import spine_row_to_dict

    return pack_dict(spine_row_to_dict(np.asarray(spine_row)))


def observation_dict_to_row(obs: dict) -> np.ndarray:
    """Spine observation dictionary (e.g. unpacked from a spine log) -> flat row ``[62]`` for the observer and
    controller pipelines; entries the dictionary lacks stay 0."""
    A = _abi
    r = np.zeros(A.SPINE_DIM, dtype=np.float32)
    bo = obs.get("base_orientation", {})
    if "angular_velocity" in bo:
        r[A.SP_BASE_ANGVEL:A.SP_BASE_ANGVEL + 3] = bo["angular_velocity"]
    if "linear_velocity" in bo:
        r[A.SP_BASE_LINVEL:A.SP_BASE_LINVEL + 3] = bo["linear_velocity"]
    if "pitch" in bo:
        r[A.SP_PITCH] = bo["pitch"]
    if "rotation_base_to_world" in bo:
        r[A.SP_ROT:A.SP_ROT + 9] = np.asarray(bo["rotation_base_to_world"], dtype=np.float32).reshape(9)
    imu = obs.get("imu", {})
    for key, off, n in (("orientation", A.SP_IMU_QUAT, 4), ("angular_velocity", A.SP_IMU_ANGVEL, 3),
                        ("linear_acceleration", A.SP_IMU_LINACC, 3), ("raw_linear_acceleration", A.SP_IMU_RAWACC, 3)):
        if key in imu:
            r[off:off + n] = imu[key]
    r[A.SP_CONTACT] = 1.0 if obs.get("floor_contact", {}).get("contact", False) else 0.0
    for j, name in enumerate(A.JOINT_NAMES):
        so = obs.get("servo", {}).get(name, {})
        for k, key in enumerate(A.OBS_KEYS):
            if key in so:
                r[A.SP_SERVO + j * 5 + k] = so[key]
    wo = obs.get("wheel_odometry", {})
    r[A.SP_ODOM_POS] = wo.get("position", 0.0)
    r[A.SP_ODOM_VEL] = wo.get("velocity", 0.0)
    return r
