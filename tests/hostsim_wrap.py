# SPDX-License-Identifier: Apache-2.0
"""ctypes wrapper of tests/hostsim/libhostsim.so (TEST INFRASTRUCTURE).

Runs the kernels' per-robot arithmetic (upkie_b200/csrc/sim_core.cuh and
mpc_core.cuh, the exact __host__ __device__ code the sm_90a kernels inline) on
the CPU so that `pytest -m "not gpu"` can check the fp32 formulation against the
fp64 oracle without a GPU. The product never loads this library.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from upkie_b200 import _abi

_HERE = os.path.join(os.path.dirname(os.path.abspath(__file__)), "hostsim")
_LIB = os.path.join(_HERE, "libhostsim.so")
_lib = None
fp = C.POINTER(C.c_float)
dp = C.POINTER(C.c_double)
u8p = C.POINTER(C.c_uint8)


def build():
    src = os.path.join(_HERE, "hostsim.cpp")
    csrc = os.path.join(os.path.dirname(_HERE), "..", "upkie_b200", "csrc")
    deps = [src] + [os.path.join(csrc, f) for f in ("sim_core.cuh", "sim_pair.cuh", "params.h", "mpc_core.cuh", "controllers_core.cuh", "observers_core.cuh")]
    if not os.path.exists(_LIB) or os.path.getmtime(_LIB) < max(os.path.getmtime(d) for d in deps):
        subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-shared", "-x", "c++", "-o", _LIB, src])
    return _LIB


def lib():
    global _lib
    if _lib is None:
        build()
        L = C.CDLL(_LIB)
        L.hostsim_create.restype = C.c_void_p
        L.hostsim_set_scalar_legs.argtypes = [C.c_void_p, C.c_int]
        L.hostsim_create.argtypes = [C.POINTER(_abi.UpkieModel), C.POINTER(_abi.UpkieSimConfig)]
        L.hostsim_destroy.argtypes = [C.c_void_p]
        L.hostsim_reset.argtypes = [C.c_void_p, C.c_int, fp, fp, fp, fp]
        L.hostsim_step_servos.argtypes = [C.c_void_p, C.c_int, fp, fp, fp, fp, fp, C.POINTER(C.c_uint32)]
        L.hostsim_step_gyropod.argtypes = [C.c_void_p, C.c_int, fp, fp, C.c_int, fp, u8p]
        L.hostsim_set_vote_always.argtypes = [C.c_int]
        L.hostsim_step_servos_rec.argtypes = [C.c_void_p, C.c_int, fp, fp, fp, fp, fp, fp]
        L.hostsim_substep.argtypes = [C.c_void_p, C.c_int, fp, fp]
        L.hostsim_spine_obs.argtypes = [C.c_void_p, C.c_int, fp, fp]
        L.hostsim_spine_obs_with_uncertainty.argtypes = [C.c_void_p, C.c_int, fp, C.c_uint32, C.c_uint64, fp]
        L.hostsim_sample_init.argtypes = [C.c_void_p, C.c_int, C.c_uint64, C.c_uint64, C.c_uint64, fp]
        L.hostsim_philox.argtypes = [C.c_uint64, C.c_uint64, C.c_uint64, C.POINTER(C.c_uint32)]
        L.hostsim_step_servos_ext.argtypes = [C.c_void_p, C.c_int, fp, fp, fp, C.c_uint32, fp]
        L.hostsim_wheel_balancer_step.argtypes = [C.POINTER(_abi.UpkieWheelBalancerConfig), C.c_int, fp, fp, fp, fp]
        L.hostsim_gaussian8.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, C.c_uint32, fp]
        L.hostsim_step_servos_noise.argtypes = [C.c_void_p, C.c_int, fp, fp, C.c_uint32, C.c_uint64, fp]
        L.hostsim_reset_spine.argtypes = [C.c_void_p, C.c_int, fp, fp, fp, fp]
        L.hostsim_step_servos_spine.argtypes = [C.c_void_p, C.c_int, fp, fp, fp, fp]
        for name in ("hostsim_mpc_step_f32", "hostsim_mpc_step_f64"):
            getattr(L, name).argtypes = [
                C.POINTER(_abi.UpkieMpcConfig), C.c_int, dp, dp, u8p, C.c_double, dp, dp, u8p, C.POINTER(C.c_int),
            ]
        _lib = L
    return _lib


def _f(a):
    return a.ctypes.data_as(fp)


class HostSim:
    """fp32 kernel arithmetic, one robot after the other, on the CPU."""

    def __init__(self, model, config, n, scalar_legs=False):
        """``scalar_legs=False``: ``step_servos`` / ``step_gyropod`` run the substep the kernels run (paired
        legs, sim_pair.cuh); ``True``: the scalar-leg variant of sim_core.cuh (``UPKIE_PAIRED_LEGS=0`` builds)."""
        self.n = n
        self._m = model.to_struct()
        self._c = config
        self._h = lib().hostsim_create(C.byref(self._m), C.byref(config))
        assert self._h, "hostsim_create failed (model not supported by the kernels)"
        lib().hostsim_set_scalar_legs(self._h, 1 if scalar_legs else 0)
        self.state = np.zeros((n, _abi.STATE_DIM), dtype=np.float32)
        self.state[:, 2] = config.init_position[2]
        self.state[:, 3] = 1.0
        self.eps = None
        self.mu = None

    def __del__(self):
        try:
            lib().hostsim_destroy(self._h)
        except Exception:
            pass

    def set_state(self, st):
        self.state = np.ascontiguousarray(st, dtype=np.float32).copy()

    def set_randomization(self, friction=None, inertia_eps=None):
        self.mu = None if friction is None else np.ascontiguousarray(friction, dtype=np.float32)
        self.eps = None if inertia_eps is None else np.ascontiguousarray(inertia_eps, dtype=np.float32)

    def _opt(self, a):
        return _f(a) if a is not None else None

    def reset(self, init):
        init = np.ascontiguousarray(init, dtype=np.float32)
        lib().hostsim_reset(self._h, self.n, _f(self.state), _f(init), self._opt(self.eps), self._opt(self.mu))

    def step_servos(self, action):
        a = np.ascontiguousarray(action, dtype=np.float32).reshape(self.n, 36)
        obs = np.empty((self.n, 6, 5), dtype=np.float32)
        err = np.zeros(self.n, dtype=np.uint32)
        lib().hostsim_step_servos(self._h, self.n, _f(self.state), _f(a), _f(obs), self._opt(self.eps),
                                  self._opt(self.mu), err.ctypes.data_as(C.POINTER(C.c_uint32)))
        return obs, err

    def step_servos_rec(self, action):
        """One tick; also returns the body-ground contact record of its last substep ``[n, BODY_REC_DIM]``."""
        a = np.ascontiguousarray(action, dtype=np.float32).reshape(self.n, 36)
        obs = np.empty((self.n, 6, 5), dtype=np.float32)
        rec = np.zeros((self.n, _abi.BODY_REC_DIM), dtype=np.float32)
        lib().hostsim_step_servos_rec(self._h, self.n, _f(self.state), _f(a), _f(obs), self._opt(self.eps),
                                      self._opt(self.mu), _f(rec))
        return obs, rec

    def step_servos_ext(self, action, ext, local_mask=0):
        """One tick under external forces ``ext[n, 7, 3]`` (newtons at the bodies' centres of mass)."""
        a = np.ascontiguousarray(action, dtype=np.float32).reshape(self.n, 36)
        e = np.ascontiguousarray(ext, dtype=np.float32).reshape(self.n, 21)
        obs = np.empty((self.n, 6, 5), dtype=np.float32)
        lib().hostsim_step_servos_ext(self._h, self.n, _f(self.state), _f(a), _f(e), int(local_mask), _f(obs))
        return obs

    def step_servos_noise(self, action, tick, env_offset=0):
        """One tick with the torque noise models, keyed like k_step<.., NOISE=1> at per-env tick ``tick``."""
        a = np.ascontiguousarray(action, dtype=np.float32).reshape(self.n, 36)
        obs = np.empty((self.n, 6, 5), dtype=np.float32)
        lib().hostsim_step_servos_noise(self._h, self.n, _f(self.state), _f(a), tick, env_offset, _f(obs))
        return obs

    def step_gyropod(self, action, act_dim):
        a = np.ascontiguousarray(action, dtype=np.float32).reshape(self.n, act_dim)
        obs6 = np.empty((self.n, 6), dtype=np.float32)
        term = np.zeros(self.n, dtype=np.uint8)
        lib().hostsim_step_gyropod(self._h, self.n, _f(self.state), _f(a), act_dim, _f(obs6), term.ctypes.data_as(u8p))
        return obs6, term

    def substep(self, tau):
        t = np.ascontiguousarray(tau, dtype=np.float32).reshape(self.n, 6)
        lib().hostsim_substep(self._h, self.n, _f(self.state), _f(t))

    def spine_obs(self):
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        lib().hostsim_spine_obs(self._h, self.n, _f(self.state), _f(out))
        return out

    def spine_obs_with_uncertainty(self, tick, env_offset=0):
        """``k_spine_obs``: torque measurement noise and ImuUncertainty included (draws of env tick ``tick``)."""
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        lib().hostsim_spine_obs_with_uncertainty(
            self._h, self.n, _f(self.state), tick, env_offset, _f(out))
        return out

    def reset_spine(self, init):
        """Spine mode: three stopped cycles from ``init[n, 25]``; returns the assembled observation rows."""
        init = np.ascontiguousarray(init, dtype=np.float32)
        if getattr(self, "lag", None) is None:
            self.lag = np.zeros((self.n, _abi.LAG_DIM), dtype=np.float32)
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        lib().hostsim_reset_spine(self._h, self.n, _f(self.state), _f(self.lag), _f(init), _f(out))
        return out

    def step_servos_spine(self, action):
        a = np.ascontiguousarray(action, dtype=np.float32).reshape(self.n, 36)
        out = np.empty((self.n, _abi.SPINE_DIM), dtype=np.float32)
        lib().hostsim_step_servos_spine(self._h, self.n, _f(self.state), _f(self.lag), _f(a), _f(out))
        return out

    def sample_init(self, seed, env_offset=0, episode=1):
        out = np.empty((self.n, _abi.INIT_DIM), dtype=np.float32)
        lib().hostsim_sample_init(self._h, self.n, seed, env_offset, episode, _f(out))
        return out


def philox(counter_lo, counter_hi, key):
    out = (C.c_uint32 * 4)()
    lib().hostsim_philox(counter_lo, counter_hi, key, out)
    return list(out)


def wheel_balancer_step(config, state, obs3, target, action):
    """fp32 kernel arithmetic of the wheel_balancer pipeline; ``state[n, 4]`` and ``action[n, 6, 6]`` in place."""
    n = state.shape[0]
    o = np.ascontiguousarray(obs3, dtype=np.float32)
    t = None if target is None else np.ascontiguousarray(target, dtype=np.float32)
    lib().hostsim_wheel_balancer_step(C.byref(config), n, _f(state), _f(o), _f(t) if t is not None else None, _f(action))


def gaussian8(seed, env, tick, slot):
    out = np.empty(8, dtype=np.float32)
    lib().hostsim_gaussian8(seed, env, tick, slot, _f(out))
    return out


def mpc_step(config, x0, v_target, contact, dt, v_cmd, double=False):
    n = x0.shape[0]
    N = int(config.nb_timesteps)
    x = np.ascontiguousarray(x0, dtype=np.float64)
    vt = np.ascontiguousarray(v_target, dtype=np.float64)
    vc = np.ascontiguousarray(v_cmd, dtype=np.float64).copy()
    plan = np.zeros((n, N))
    found = np.zeros(n, dtype=np.uint8)
    iters = np.zeros(n, dtype=np.int32)
    c = None if contact is None else np.ascontiguousarray(contact, dtype=np.uint8)
    fn = lib().hostsim_mpc_step_f64 if double else lib().hostsim_mpc_step_f32
    fn(C.byref(config), n, x.ctypes.data_as(dp), vt.ctypes.data_as(dp), c.ctypes.data_as(u8p) if c is not None else None,
       float(dt), vc.ctypes.data_as(dp), plan.ctypes.data_as(dp), found.ctypes.data_as(u8p),
       iters.ctypes.data_as(C.POINTER(C.c_int)))
    return vc, plan, found, iters
