# SPDX-License-Identifier: Apache-2.0
"""ctypes loader of ``libupkie_b200.so`` (the C ABI of ``include/upkie_b200.h``).

The library is built in-tree by ``upkie_b200.build.build()`` (nvcc, sm_90a). There
is no fallback: if the shared object is missing, or no CUDA device is present
when a handle is created, the product path raises.
"""

import ctypes as C
import os

from . import _abi
from .exceptions import MissingOptionalDependency, UpkieRuntimeError

_HERE = os.path.dirname(os.path.abspath(__file__))
# UPKIE_B200_LIB: developer override used by tools/variants.py to load an alternative build
LIB_PATH = os.environ.get("UPKIE_B200_LIB") or os.path.join(_HERE, "libupkie_b200.so")

_lib = None

_fp = C.POINTER(C.c_float)
_u8p = C.POINTER(C.c_uint8)
_vp = C.c_void_p

# name -> (restype, argtypes); every symbol include/upkie_b200.h declares
SYMBOLS = {
    "upkie_b200_abi_version": (C.c_int, []),
    "upkie_b200_last_error": (C.c_char_p, []),
    "upkie_b200_default_config": (C.c_int, [C.POINTER(_abi.UpkieSimConfig)]),
    "upkie_b200_default_mpc_config": (C.c_int, [C.POINTER(_abi.UpkieMpcConfig)]),
    "upkie_b200_create": (
        C.c_int,
        [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig), C.c_int, C.c_int, C.POINTER(_vp)],
    ),
    "upkie_b200_destroy": (None, [_vp]),
    "upkie_b200_num_envs": (C.c_int, [_vp]),
    "upkie_b200_set_autoreset": (C.c_int, [_vp, C.c_int, C.c_uint64, C.c_uint64]),
    "upkie_b200_set_config": (C.c_int, [_vp, C.POINTER(_abi.UpkieSimConfig)]),
    "upkie_b200_set_randomization": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_env_params": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_get_env_params": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_get_randomization": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_reset_randomization": (C.c_int, [_vp, C.POINTER(_abi.UpkieResetRandomization)]),
    "upkie_b200_get_draws": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_draws": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_push_randomization": (C.c_int, [_vp, C.POINTER(_abi.UpkiePushRandomization)]),
    "upkie_b200_get_push_forces": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_get_push_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_push_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_action_delay": (C.c_int, [_vp, C.POINTER(_abi.UpkieActionDelay)]),
    "upkie_b200_get_action_delay_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_action_delay_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_observation_delay": (C.c_int, [_vp, C.POINTER(_abi.UpkieObservationDelay)]),
    "upkie_b200_get_observation_delay_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_observation_delay_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_action_delay_ticks": (C.c_int, [_vp, C.POINTER(_abi.UpkieActionDelay), C.c_uint32]),
    "upkie_b200_get_action_delay_history": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_action_delay_history": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_observation_delay_ticks": (C.c_int, [_vp, C.POINTER(_abi.UpkieObservationDelay), C.c_uint32]),
    "upkie_b200_get_observation_delay_history": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_observation_delay_history": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_servo_dropout": (C.c_int, [_vp, C.POINTER(_abi.UpkieServoDropout)]),
    "upkie_b200_get_servo_dropout_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_servo_dropout_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_imu_misalignment": (C.c_int, [_vp, C.POINTER(_abi.UpkieImuMisalignment)]),
    "upkie_b200_get_imu_misalignment_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_imu_misalignment_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_encoder_offset": (C.c_int, [_vp, C.POINTER(_abi.UpkieEncoderOffset)]),
    "upkie_b200_get_encoder_offset_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_encoder_offset_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_servo_noise": (C.c_int, [_vp, C.POINTER(_abi.UpkieServoNoise)]),
    "upkie_b200_get_servo_noise_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_servo_noise_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_get_servo_noise_mark": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_servo_noise_mark": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_velocity_derate": (C.c_int, [_vp, C.POINTER(_abi.UpkieVelocityDerate)]),
    "upkie_b200_get_velocity_derate_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_velocity_derate_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_attitude_filter": (C.c_int, [_vp, C.POINTER(_abi.UpkieAttitudeFilter)]),
    "upkie_b200_get_attitude_filter_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_attitude_filter_state": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_get_attitude_filter_report": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_attitude_filter_report": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_torque_scale": (C.c_int, [_vp, C.POINTER(_abi.UpkieTorqueScale)]),
    "upkie_b200_get_torque_scale_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_torque_scale_state": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_set_history": (C.c_int, [_vp, C.POINTER(_abi.UpkieHistory)]),
    "upkie_b200_get_history": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_history_entries": (C.c_int, [_vp, C.POINTER(C.c_int)]),
    "upkie_b200_get_history_state": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_history_state": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_reset": (C.c_int, [_vp, _vp, _vp, C.c_uint64, C.c_uint64, _vp]),
    "upkie_b200_step_servos": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_step_gyropod": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_step_servos_compact": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_step_servos_multicast": (C.c_int, [_vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_step_servos_peers": (C.c_int, [_vp, _vp, _vp, _vp, C.c_int, _vp]),
    "upkie_b200_step_servos_push": (C.c_int, [_vp, _vp, _vp, _vp, C.POINTER(_abi.UpkiePush), _vp]),
    "upkie_b200_push_rows": (C.c_int, [_vp, C.POINTER(_abi.UpkiePush), _vp]),
    "upkie_b200_step_servos_host": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_step_gyropod_host": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp, _vp]),
    "upkie_b200_step_servos_host_compact": (C.c_int, [_vp, _vp, _vp, _vp]),
    "upkie_b200_step": (C.c_int, [_vp, C.c_int, _vp, C.POINTER(_abi.UpkieStepOutputs), _vp]),
    "upkie_b200_step_host": (C.c_int, [_vp, C.c_int, _vp, C.POINTER(_abi.UpkieStepOutputs)]),
    "upkie_b200_spine_obs": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_final_spine_obs": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_reset_obs": (C.c_int, [_vp, C.c_int, _vp, _vp]),
    "upkie_b200_get_state": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_get_lag": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_get_body_contacts": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_lag": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_state": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_error_flags": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_get_counters": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_set_counters": (C.c_int, [_vp, _vp, _vp, _vp, _vp, _vp]),
    "upkie_b200_get_elapsed": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_elapsed": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_set_external_forces": (C.c_int, [_vp, _vp, C.c_uint32, _vp]),
    "upkie_b200_default_wheel_balancer_config": (C.c_int, [_vp]),
    "upkie_b200_wheel_balancer_create": (C.c_int, [_vp, C.c_int, C.c_int, C.POINTER(C.c_void_p)]),
    "upkie_b200_wheel_balancer_destroy": (None, [_vp]),
    "upkie_b200_wheel_balancer_reset": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_wheel_balancer_step": (C.c_int, [_vp, _vp, C.c_int, _vp, _vp, _vp]),
    "upkie_b200_wheel_balancer_state": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_launch_count": (C.c_int, [_vp, C.POINTER(C.c_uint64)]),
    "upkie_b200_mpc_create": (C.c_int, [C.POINTER(_abi.UpkieMpcConfig), C.c_int, C.c_int, C.POINTER(_vp)]),
    "upkie_b200_mpc_destroy": (None, [_vp]),
    "upkie_b200_mpc_reset": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_mpc_step": (C.c_int, [_vp, _vp, _vp, _vp, C.c_float, _vp, _vp, _vp, _vp]),
    "upkie_b200_mpc_plan": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_base_velocity_post": (C.c_int, [_vp, _vp, C.POINTER(_abi.UpkieBaseVelocityPost), _vp]),
    "upkie_b200_default_observer_config": (C.c_int, [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieObserverConfig)]),
    "upkie_b200_observers_create": (C.c_int, [C.POINTER(_abi.UpkieObserverConfig), C.c_int, C.c_int, C.POINTER(_vp)]),
    "upkie_b200_observers_destroy": (None, [_vp]),
    "upkie_b200_observers_reset": (C.c_int, [_vp, _vp, _vp]),
    "upkie_b200_observers_step": (C.c_int, [_vp, _vp, _vp, _vp]),
}


def lib():
    """Load the shared library (once). Raises if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise MissingOptionalDependency(
                f"{LIB_PATH} not found: build it with "
                "`python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). upkie_b200 has no CPU fallback."
            )
        L = C.CDLL(LIB_PATH)
        for name, (restype, argtypes) in SYMBOLS.items():
            fn = getattr(L, name)  # AttributeError if the .so lacks a declared symbol
            fn.restype = restype
            fn.argtypes = argtypes
        if L.upkie_b200_abi_version() != _abi.ABI_VERSION:
            raise UpkieRuntimeError(
                f"libupkie_b200.so ABI {L.upkie_b200_abi_version()} != {_abi.ABI_VERSION}"
            )
        _lib = L
    return _lib


def check(rc: int) -> None:
    """Turn a C status code into the reference's exception types
    (``upkie/exceptions.py``)."""
    if rc == 0:
        return
    msg = lib().upkie_b200_last_error().decode("utf-8", "replace")
    raise UpkieRuntimeError(f"libupkie_b200 error {rc}: {msg}")
