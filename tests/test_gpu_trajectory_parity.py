# SPDX-License-Identifier: Apache-2.0
"""Trajectory parity on the device: the fast-math step kernels against the fp64 oracle over closed-loop rollouts.

The one-tick tests (test_gpu_sim_parity.py, test_gpu_exact_mode.py) start every side from the same state. Here each
side closes its loop on its OWN observations for 400 ticks (2 s), never re-synchronised: the device on the path under
test, the fp64 oracle, the oracle in fp32, the kernels' arithmetic compiled for the host (tests/hostsim) and, where
the kernel family exists there, the library built without --use_fast_math. What fp32 alone costs is what the host
build and the fp32 oracle drift; the device may not drift an order of magnitude more. Measured drifts go to the JSON
file named by UPKIE_PARITY_REPORT."""
import ctypes as C
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from upkie_b200 import _abi

pytestmark = pytest.mark.gpu

N = 1027  # neither a whole warp nor a whole 256-thread block
TICKS = 400
EVERY = 50
CAP_PITCH = 1e-4  # rad, as tests/test_kernel_arithmetic_cpu.py's two-second loop
CAP_POS = 5e-4  # m, ground position
# The device may drift at most RATIO x as far as the worst of the fp32 sides that run without fast math (host build,
# fp32 oracle, exact library), plus a floor. Measured on an H100: 1.5x at worst with the polynomial integrator; 3.3x to
# 10.7x with the fast-math sinf / cosf it replaced; 2.6x to 3.7x with a 1e-4 relative error in the rotation increment.
RATIO = 2.5
FLOOR_PITCH, FLOOR_POS, FLOOR_YAW = 2e-6, 1e-5, 1e-5
SQUAT = (100, 200, 300)  # knee targets ramp out, sit 0.05 rad past the bound for 0.5 s, ramp back
THREADS = os.cpu_count() or 1
SPIN_FLOOR = 1e-9  # rad after 200 ticks of free spin from the identity


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _report(name, **values):
    from test_gpu_sim_parity import _report as report

    report(name, **values)


# -- state-row quantities (fp64) ------------------------------------------------------------------------------------
def _pitch(st):
    w, x, y, z = st[:, 3], st[:, 4], st[:, 5], st[:, 6]
    return np.arcsin(np.clip(2.0 * (w * y - z * x), -1.0, 1.0))  # base_pitch of sim_core.cuh


def _yaw(st):
    w, x, y, z = st[:, 3], st[:, 4], st[:, 5], st[:, 6]
    return np.arctan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z))


def _ground(model, st, col):
    """Ground position (``col`` = ST_Q) or velocity (``col`` = ST_QD) from the wheel angles or rates."""
    sign = 1.0 if model.left_wheeled else -1.0
    return 0.5 * (st[:, col + 2] - st[:, col + 5]) * sign * float(model.wheel_radius)


def _angle_between(qa, qb):
    """Rotation angle of qa^-1 qb, accurate for small angles."""
    w = np.abs(np.sum(qa * qb, axis=1))
    cross = np.linalg.norm(qa[:, :1] * qb[:, 1:] - qb[:, :1] * qa[:, 1:] - np.cross(qa[:, 1:], qb[:, 1:]), axis=1)
    return 2.0 * np.arctan2(cross, w)


def _wrap(a):
    return (a + np.pi) % (2.0 * np.pi) - np.pi


# -- policies -------------------------------------------------------------------------------------------------------
def _pd(pitch, pos, vel):
    """README PD policy (gains of test_kernel_arithmetic_cpu.py's two-second loop): ground velocity command."""
    return 10.0 * pitch + 1.0 * pos + 0.1 * vel


def _knee_target(model, t, squat):
    """``squat = (ramp, hold, back)`` ticks: knee targets ramp out until ``ramp``, stay 0.05 rad past the bound until
    ``hold`` and ramp back until ``back``; None holds the legs straight."""
    if squat is None:
        return 0.0
    top = model.joints[1].limit.upper + 0.05
    ramp, hold, back = squat
    if t < ramp:
        return top * t / ramp
    if t < hold:
        return top
    return top * max(back - t, 0) / (back - hold)


def _servo_action(model, st, knee):
    """UpkieServos action rows from a side's own state row: the PD on the wheels as velocity targets (NaN position),
    the legs held in position, knees at +-``knee`` and hips at -+``knee / 2`` so the wheels stay under the hips."""
    st = st.astype(np.float64)
    n = st.shape[0]
    gv = _pd(_pitch(st), _ground(model, st, _abi.ST_Q), _ground(model, st, _abi.ST_QD))
    sign = 1.0 if model.left_wheeled else -1.0
    a = np.zeros((n, 6, 6), dtype=np.float32)
    a[:, :, 3] = a[:, :, 4] = 1.0
    a[:, :, 5] = np.asarray(model.tau_max, dtype=np.float32)
    a[:, [2, 5], 0] = np.nan
    a[:, 2, 1] = sign * gv / float(model.wheel_radius)
    a[:, 5, 1] = -sign * gv / float(model.wheel_radius)
    a[:, 0, 0], a[:, 1, 0], a[:, 3, 0], a[:, 4, 0] = 0.5 * knee, -knee, -0.5 * knee, knee
    return a


# -- the sides ------------------------------------------------------------------------------------------------------
class _Oracle:
    def __init__(self, oracle_lib, model, cfg, n, use_float):
        self.s = oracle_lib.OracleSim(model, cfg, n, use_float=use_float, threads=THREADS)

    def randomize(self, mu, eps):
        self.s.set_randomization(friction=mu.astype(np.float64), inertia_eps=eps.astype(np.float64))

    def reset(self, init):
        self.s.reset(init.astype(np.float64))

    def set_state(self, st):
        self.s.set_state(st.astype(np.float64))

    def gyro(self, a):
        o, _, term, _ = self.s.step_gyropod(a.astype(np.float64), a.shape[1])
        return o, term

    def servos(self, a):
        return self.s.step_servos(a.astype(np.float64))[2]

    def state(self):
        return self.s.get_state()


class _Host:
    """The host build, its robots split over threads (ctypes releases the GIL; the robots are independent)."""

    def __init__(self, model, cfg, n):
        from hostsim_wrap import HostSim

        k = max(1, min(THREADS, n // 64))
        self.cuts = np.linspace(0, n, k + 1).astype(int)
        self.parts = [HostSim(model, cfg, int(b - a)) for a, b in zip(self.cuts[:-1], self.cuts[1:])]
        self.pool = ThreadPoolExecutor(len(self.parts))

    def _each(self, fn, *arrays):
        jobs = [self.pool.submit(fn, p, *[x[a:b] for x in arrays])
                for p, a, b in zip(self.parts, self.cuts[:-1], self.cuts[1:])]
        return [j.result() for j in jobs]

    def randomize(self, mu, eps):
        self._each(lambda p, m, e: p.set_randomization(m, e), mu, eps)

    def reset(self, init):
        self._each(lambda p, i: p.reset(i), init)

    def set_state(self, st):
        self._each(lambda p, s: p.set_state(s), st)

    def gyro(self, a):
        out = self._each(lambda p, x: p.step_gyropod(x, a.shape[1]), a)
        o6, term = np.concatenate([o for o, _ in out]), np.concatenate([t for _, t in out])
        # pendulum: the oracle's and the device's [pitch, ground position, angular velocity, ground velocity]
        return (o6 if a.shape[1] == 2 else o6[:, [1, 0, 4, 3]]), term

    def servos(self, a):
        self._each(lambda p, x: p.step_servos(x), a)
        return None  # the host build has no termination logic for UpkieServos

    def state(self):
        return np.concatenate([p.state for p in self.parts]).astype(np.float64)

    def close(self):
        self.pool.shutdown()


class _Device:
    """A handle of the product library on one step path."""

    def __init__(self, torch, model, cfg, n, path):
        from upkie_b200.sim import UpkieSim

        self.torch, self.path = torch, path
        self.sim = UpkieSim(n, model=model, config=cfg)
        if path == "compact":
            self.sim.set_autoreset(1, 2025, 0)  # the headline's next-step auto-reset
        if path in ("gyropod_host",):
            self.buf = self.sim.host_action_buffer(2)

    def _t(self, x):
        return self.torch.from_numpy(np.ascontiguousarray(x)).cuda()

    def randomize(self, mu, eps):
        self.sim.set_randomization(friction=self._t(mu), inertia_eps=self._t(eps))

    def reset(self, init):
        self.sim.reset(init_state=self._t(init))
        if self.path == "table":  # a table equal to the config: the FAM_TABLE kernels, the same physics
            self.sim.set_env_params(self.sim.get_env_params())

    def set_state(self, st):
        self.sim.set_state(self._t(st.astype(np.float32)))

    def gyro(self, a):
        if self.path == "gyropod_host":
            self.buf[:] = a
            o, _, term, _ = self.sim.step_gyropod_host(self.buf)
            return o.astype(np.float64), term.copy()
        step = self.sim.step_pendulum if a.shape[1] == 1 else self.sim.step_gyropod
        o, _, term, _ = step(self._t(a))
        return o.cpu().numpy().astype(np.float64), term.cpu().numpy()

    def servos(self, a):
        if self.path == "compact":
            return self.sim.step_servos_compact(self._t(a))[1].cpu().numpy()
        return self.sim.step_servos(self._t(a))[2].cpu().numpy()

    def state(self):
        return self.sim.get_state().cpu().numpy().astype(np.float64)


class _Exact:
    """The library built without --use_fast_math (device buffers, TILE = 0), through its C ABI."""

    def __init__(self, torch, model, cfg, n):
        from test_gpu_exact_mode import _load_exact

        self.L, self.torch, self.n = _load_exact(), torch, n
        self._m, self._c = model.to_struct(), cfg
        self.h = C.c_void_p()
        assert self.L.upkie_b200_create(C.byref(self._m), C.byref(self._c), n, 0, C.byref(self.h)) == 0
        dev = torch.device("cuda", 0)
        self.s = C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)
        z = lambda *shape, dt=torch.float32: torch.empty(shape, dtype=dt, device=dev)  # noqa: E731
        self.obs30, self.obs6, self.obs4 = z(n, 6, 5), z(n, 6), z(n, 4)
        self.rew, self.term, self.trunc = z(n), z(n, dt=torch.uint8), z(n, dt=torch.uint8)
        self.st = z(n, _abi.STATE_DIM)
        self.keep = []

    def _p(self, x):
        t = x if hasattr(x, "data_ptr") else self.torch.from_numpy(np.ascontiguousarray(x)).cuda()
        self.keep = [t]
        return C.c_void_p(t.data_ptr())

    def _ok(self, rc):
        assert rc == 0, self.L.upkie_b200_last_error()

    def randomize(self, mu, eps):
        m, e = self.torch.from_numpy(mu).cuda(), self.torch.from_numpy(eps).cuda()
        self._ok(self.L.upkie_b200_set_randomization(self.h, C.c_void_p(m.data_ptr()), C.c_void_p(e.data_ptr()), self.s))
        self.torch.cuda.synchronize()

    def reset(self, init):
        self._ok(self.L.upkie_b200_reset(self.h, None, self._p(init), 0, 0, self.s))

    def set_state(self, st):
        self._ok(self.L.upkie_b200_set_state(self.h, self._p(st.astype(np.float32)), self.s))

    def gyro(self, a):
        obs = self.obs6 if a.shape[1] == 2 else self.obs4
        self._ok(self.L.upkie_b200_step_gyropod(self.h, self._p(a), a.shape[1], C.c_void_p(obs.data_ptr()),
                                                C.c_void_p(self.rew.data_ptr()), C.c_void_p(self.term.data_ptr()),
                                                C.c_void_p(self.trunc.data_ptr()), self.s))
        return obs.cpu().numpy().astype(np.float64), self.term.cpu().numpy()

    def servos(self, a):
        self._ok(self.L.upkie_b200_step_servos(self.h, self._p(a), C.c_void_p(self.obs30.data_ptr()),
                                               C.c_void_p(self.rew.data_ptr()), C.c_void_p(self.term.data_ptr()),
                                               C.c_void_p(self.trunc.data_ptr()), self.s))
        return self.term.cpu().numpy()

    def state(self):
        self._ok(self.L.upkie_b200_get_state(self.h, C.c_void_p(self.st.data_ptr()), self.s))
        self.torch.cuda.synchronize()
        return self.st.cpu().numpy().astype(np.float64)

    def close(self):
        self.L.upkie_b200_destroy(self.h)


# -- closed-loop runner ---------------------------------------------------------------------------------------------
CONFIG_KEYS = ("joint_limits", "body", "overrides")


def _config(kind, joint_limits=3, body=0, overrides=()):
    """``overrides``: ``(field, value)`` pairs of UpkieSimConfig set last, e.g. ``(("dt", 0.01), ("nb_substeps", 10))``
    (a tuple, so that it keys the reference cache)."""
    cfg = _abi.default_sim_config()
    if kind == "servos":  # the headline workload's termination (bench.py: servos_config)
        cfg.servos_fall_termination, cfg.min_base_height = 1, 0.15
        cfg.joint_limits, cfg.body_contacts = joint_limits, body
    for k, v in overrides:
        setattr(cfg, k, v)
    return cfg


def _initial(n, seed=0, crouch=False):
    """Initial pitches in +-0.25 rad; ``crouch``: knees 0.01 rad inside their bound, the base lowered to match."""
    rng = np.random.default_rng(seed)
    pitch = rng.uniform(-0.25, 0.25, n)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2], init[:, 3], init[:, 5] = 0.6, np.cos(pitch / 2), np.sin(pitch / 2)
    if crouch:
        init[:, 2] = 0.345
        init[:, _abi.ST_Q:_abi.ST_Q + 6] = np.array([1.25, -2.5, 0.0, -1.25, 2.5, 0.0], dtype=np.float32)
    mu = rng.uniform(0.5, 1.2, n).astype(np.float32)
    eps = rng.uniform(-0.2, 0.2, (n, 6)).astype(np.float32)
    return init, mu, eps


def _rollout(model, sides, kind, n, ticks, squat=None, yaw_rate=None, seed=0, crouch=False):
    """Every side runs its own closed loop. Returns per side ``(states, terminated)``: the state rows after every
    ``EVERY``-th tick, fp64 ``[ticks // EVERY, n, STATE_DIM]``, and ``terminated`` of every tick ``[ticks, n]`` (None
    where a side does not compute it). Servos runs carry the headline's randomisation: floor friction in [0.5, 1.2],
    inertia epsilons in +-0.2, the same on every side."""
    init, mu, eps = _initial(n, seed, crouch)
    for s in sides.values():
        if kind == "servos":
            s.randomize(mu, eps)
        s.reset(init)
    obs = {k: np.zeros((n, 6 if kind == "gyropod" else 4)) for k in sides}
    states = {k: [] for k in sides}
    terms = {k: [] for k in sides}
    for t in range(ticks):
        for k, s in sides.items():
            if kind == "servos":
                term = s.servos(_servo_action(model, s.state(), _knee_target(model, t, squat)))
            elif kind == "gyropod":
                o = obs[k]
                v = _pd(o[:, 1], o[:, 0], o[:, 3])
                a = np.stack([v, np.zeros(n) if yaw_rate is None else yaw_rate], 1).astype(np.float32)
                obs[k], term = s.gyro(a)
            else:  # pendulum: [pitch, ground position, angular velocity, ground velocity]
                o = obs[k]
                obs[k], term = s.gyro(_pd(o[:, 0], o[:, 1], o[:, 3]).reshape(n, 1).astype(np.float32))
            terms[k].append(term)
            if t % EVERY == EVERY - 1:
                states[k].append(s.state())
    return {k: (np.stack(states[k]), None if terms[k][0] is None else np.stack(terms[k])) for k in sides}


_REFERENCES = {}


def _references(model, oracle_lib, torch, kind, n=N, ticks=TICKS, exact=True, **kw):
    """The sides that do not depend on the device path: fp64 and fp32 oracle, host build, exact library. Cached per
    physics, so that runs which differ only in the device path share them."""
    key = (kind, n, ticks, exact, tuple(sorted(kw.items(), key=lambda x: x[0])))
    if key not in _REFERENCES:
        cfg = _config(kind, **{k: v for k, v in kw.items() if k in CONFIG_KEYS})
        sides = {"oracle": _Oracle(oracle_lib, model, cfg, n, False), "oracle32": _Oracle(oracle_lib, model, cfg, n, True),
                 "host": _Host(model, cfg, n)}
        if exact:
            sides["exact"] = _Exact(torch, model, cfg, n)
        run_kw = {k: v for k, v in kw.items() if k in ("squat", "yaw_rate", "seed", "crouch")}
        if isinstance(run_kw.get("yaw_rate"), tuple):
            run_kw["yaw_rate"] = np.asarray(run_kw["yaw_rate"])
        _REFERENCES[key] = _rollout(model, sides, kind, n, ticks, **run_kw)
        sides["host"].close()
        if exact:
            sides["exact"].close()
    return _REFERENCES[key]


def _drift(model, a, b):
    """Worst pitch, ground-position and yaw difference and contact-flag mismatches between two runs' snapshots."""
    (sa, _), (sb, _) = a, b
    pa, pb = sa.reshape(-1, sa.shape[-1]), sb.reshape(-1, sb.shape[-1])
    return {"pitch": np.abs(_pitch(pa) - _pitch(pb)).max(),
            "pos": np.abs(_ground(model, pa, _abi.ST_Q) - _ground(model, pb, _abi.ST_Q)).max(),
            "yaw": np.abs(_wrap(_yaw(pa) - _yaw(pb))).max(),
            "contact": int((pa[:, _abi.ST_CONTACT] != pb[:, _abi.ST_CONTACT]).sum())}


def _check_run(model, name, dev, refs, caps=(CAP_PITCH, CAP_POS)):
    d = {k: _drift(model, r, refs["oracle"]) for k, r in list(refs.items()) + [("device", dev)] if k != "oracle"}
    _report(f"trajectory_{name}", **{f"{k}_{m}": v for k, e in d.items() for m, v in e.items()})
    g = d["device"]
    h = {m: max(e[m] for k, e in d.items() if k != "device") for m in ("pitch", "pos", "yaw")}  # worst fp32 side
    # terminated, tick by tick, bit for bit
    for k in ("device", "exact"):
        run = dev if k == "device" else refs.get(k)
        if run is not None and run[1] is not None:
            assert np.array_equal(run[1], refs["oracle"][1]), (name, k)
    assert g["pitch"] < caps[0] and g["pos"] < caps[1], (name, g)
    assert g["contact"] <= 1, (name, g)  # at most one robot within round-off of the breaking threshold
    assert g["pitch"] <= RATIO * h["pitch"] + FLOOR_PITCH and g["pos"] <= RATIO * h["pos"] + FLOOR_POS, (name, g, h)
    assert g["yaw"] <= RATIO * h["yaw"] + FLOOR_YAW, (name, g, h)
    for k, (st, _) in list(refs.items()) + [("device", dev)]:  # nobody fell: these are balancing robots
        assert np.abs(_pitch(st[-1])).max() < 0.5, (name, k)
    return d


# Caps: the CPU test's 1e-4 rad / 5e-4 m where the host build stays well inside them. UpkieServos runs carry the
# headline's randomisation, and there fp32 alone drifts further. Measured with the host build over these 1 027 robots:
# 9.6e-5 rad / 1.3e-4 m with straight legs, 1.8e-4 rad / 1.8e-3 m with the squat (the fp32 oracle: 7.6e-5 / 1.1e-4 and
# 2.0e-4 / 1.9e-3). Those caps are ten times the host build's drift. The gyropod at 1 000 Hz, one substep, drifts
# further in its 0.4 s than at 200 Hz in 2 s (host build 7.3e-5 rad / 1.4e-5 m, fp32 oracle 6.5e-5 / 1.3e-5): CAPS_SERVOS.
CAPS_SERVOS = (1e-3, 2e-3)
CAPS_SQUAT = (2e-3, 2e-2)
RUNS = {
    # name: (kind, device path, reference keywords, (pitch cap, ground-position cap))
    "gyropod_device": ("gyropod", "gyropod", {}, (CAP_PITCH, CAP_POS)),
    "gyropod_pinned_host": ("gyropod", "gyropod_host", {}, (CAP_PITCH, CAP_POS)),
    "pendulum": ("pendulum", "pendulum", {}, (CAP_PITCH, CAP_POS)),
    "servos_plain": ("servos", "servos", {"joint_limits": 0}, CAPS_SERVOS),
    "servos_limits2_squat": ("servos", "servos", {"joint_limits": 2, "squat": SQUAT}, CAPS_SQUAT),
    "servos_limits3_squat": ("servos", "servos", {"joint_limits": 3, "squat": SQUAT}, CAPS_SQUAT),
    "servos_headline_squat": ("servos", "compact", {"joint_limits": 3, "squat": SQUAT}, CAPS_SQUAT),
    "servos_table_squat": ("servos", "table", {"joint_limits": 3, "squat": SQUAT}, CAPS_SQUAT),
    "servos_body": ("servos", "servos", {"joint_limits": 3, "body": 1, "exact": False}, CAPS_SERVOS),
    # away from the default config (test_gpu_config_parity.py holds the same knobs to the oracle over one tick)
    "gyropod_100hz_10_substeps": ("gyropod", "gyropod", {"overrides": (("dt", 0.01), ("nb_substeps", 10))},
                                  (CAP_PITCH, CAP_POS)),
    "gyropod_1000hz_1_substep": ("gyropod", "gyropod", {"overrides": (("dt", 0.001), ("nb_substeps", 1))},
                                 CAPS_SERVOS),
    "gyropod_friction_0.3": ("gyropod", "gyropod", {"overrides": (("friction", 0.3),)}, (CAP_PITCH, CAP_POS)),
    "servos_warm_start_3_sweeps_squat": ("servos", "servos", {"joint_limits": 3, "squat": SQUAT, "overrides": (
        ("warmstarting_factor", 0.85), ("pgs_iterations", 3), ("solver_residual_threshold", 0.0))}, CAPS_SQUAT),
}


@pytest.mark.parametrize("name", list(RUNS))
def test_two_second_closed_loop_on_the_device(model, oracle_lib, torch, name):
    """400 ticks from initial pitches in +-0.25 rad: pitch and ground position within the run's caps of the fp64
    oracle every 50 ticks, `terminated` equal on every tick, and pitch, ground position and yaw drift within RATIO x
    the worst fp32 side's."""
    kind, path, kw, caps = RUNS[name]
    refs = _references(model, oracle_lib, torch, kind, **kw)
    cfg = _config(kind, **{k: v for k, v in kw.items() if k in CONFIG_KEYS})
    dev = _rollout(model, {"device": _Device(torch, model, cfg, N, path)}, kind, N, TICKS,
                   squat=kw.get("squat"))["device"]
    _check_run(model, name, dev, refs, caps)
    if kw.get("squat"):  # the knees reached their bound: the limit rows were active
        knees = dev[0][SQUAT[1] // EVERY - 1][:, [_abi.ST_Q + 1, _abi.ST_Q + 4]]
        assert np.abs(knees).min() > model.joints[1].limit.upper - 2e-3, np.abs(knees).min()


def test_turn_in_place(model, oracle_lib, torch):
    """Gyropod with a constant yaw-rate command per env, log-spaced over [1e-3, 1] rad/s: the base yaw read from the
    quaternion stays as close to the oracle's as the fp32 sides' does (within RATIO x, plus 1e-5 rad)."""
    rates = tuple(np.geomspace(1e-3, 1.0, N).astype(np.float32).tolist())
    refs = _references(model, oracle_lib, torch, "gyropod", yaw_rate=rates)
    dev = _rollout(model, {"device": _Device(torch, model, _config("gyropod"), N, "gyropod")}, "gyropod", N, TICKS,
                   yaw_rate=np.asarray(rates))["device"]
    d = _check_run(model, "turn_in_place", dev, refs)
    assert np.abs(_yaw(dev[0][-1])).max() > 0.1  # the robots did turn
    assert d["device"]["yaw"] < 1e-3


def test_slow_rotation_of_the_orientation_integrator(model, oracle_lib, torch):
    """A free-floating robot (no gravity, far above the floor, zero joint torques) spun about random axes at base
    rates from 1e-5 to 30 rad/s, both sides of the integrator's small-angle switch at 1e-3 rad/s and one fp32 ulp
    around it, for 200 ticks. The rotation between each side's base orientation and the fp64 oracle's: the fast
    library's stays within RATIO x the worst fp32 side's, decade by decade, and every quaternion stays a unit one.

    The robots start from the identity orientation. From a general one, fp32 storage of the quaternion alone rounds
    every substep's turn by up to an ulp of its components (6e-8), which at these rates is the increment itself: all
    fp32 sides then share a 5e-5 rad floor after 1 s, and an integrator error below it goes unseen. From the identity
    the small components carry the turn with full relative precision; the floor is what the arithmetic costs."""
    per = 8
    one = np.float32(1e-3)
    speeds = np.concatenate([np.geomspace(1e-5, 30.0, 28), [np.nextafter(one, np.float32(0)), one,
                                                            np.nextafter(one, np.float32(1))]])
    n = per * speeds.size
    rng = np.random.default_rng(11)
    axes = rng.normal(size=(n, 3))
    axes /= np.linalg.norm(axes, axis=1, keepdims=True)
    w = np.repeat(speeds, per)
    exact_norm = np.repeat(np.arange(speeds.size) >= 28, per)  # the ulp cases: one axis, so |omega| is exact in fp32
    axes[exact_norm] = np.eye(3)[rng.integers(0, 3, exact_norm.sum())]
    st = np.zeros((n, _abi.STATE_DIM))
    st[:, 2] = 20.0  # the base turns about its origin, not about the centre of mass: the robot flies off at up to 9 m/s
    st[:, 3] = 1.0
    st[:, _abi.ST_ANGVEL:_abi.ST_ANGVEL + 3] = axes * w[:, None]
    st = st.astype(np.float32)
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 3] = act[:, :, 4] = 1.0  # max_torque 0: no joint torque at all
    cfg = _abi.default_sim_config()
    cfg.gravity = 0.0
    sides = {"oracle": _Oracle(oracle_lib, model, cfg, n, False), "oracle32": _Oracle(oracle_lib, model, cfg, n, True),
             "host": _Host(model, cfg, n), "exact": _Exact(torch, model, cfg, n),
             "fast": _Device(torch, model, cfg, n, "servos")}
    for s in sides.values():
        s.set_state(st)
    for _ in range(200):
        for s in sides.values():
            s.servos(act)
    out = {k: s.state() for k, s in sides.items()}
    sides["host"].close()
    sides["exact"].close()
    ref = out["oracle"][:, 3:7]
    assert min(o[:, 2].min() for o in out.values()) > 5.0  # free flight all along
    err = {k: _angle_between(out[k][:, 3:7], ref) for k in ("fast", "exact", "host", "oracle32")}
    for k, o in out.items():
        assert np.abs(np.linalg.norm(o[:, 3:7], axis=1) - 1.0).max() < 1e-6, k
    decade = np.floor(np.log10(w)).astype(int)
    report = {}
    for d in np.unique(decade):
        sel = decade == d
        e = {k: v[sel].max() for k, v in err.items()}
        report.update({f"1e{d}_{k}": v for k, v in e.items()})
    _report("slow_rotation_200_ticks", **report)
    for d in np.unique(decade):
        e = {k: report[f"1e{d}_{k}"] for k in err}
        assert e["fast"] <= RATIO * max(e["exact"], e["host"], e["oracle32"]) + SPIN_FLOOR, (d, e)


@pytest.mark.parametrize("n", [1, 31, 33, 257, 4097])
def test_tail_lanes_follow_the_oracle(model, oracle_lib, torch, n):
    """Batches that end inside a warp and inside a block: the tail lanes shadow robot n - 1 and vote with their
    warp (solver paths, mode 3's per-warp limit rows), but only real robots store. 50 closed-loop ticks on the
    headline path (compact rows, TILE 1, crouched with the knee targets past their bound) and on the device-buffer
    gyropod (TILE 0); every env is compared with the fp64 oracle. Crouched on the bound, a limit row that engages one
    substep earlier or later moves a robot by more than the 400-tick caps within 50 ticks, in the host build as much
    as on the device (measured on the CPU: 2.8e-3 rad over 4 097 robots). So the cap is the host build's drift on the
    same robots, RATIO x plus a floor far below a fast-math integrator's 1e-5 rad."""
    ticks = 50
    for kind, path, kw in (("servos", "compact", {"joint_limits": 3, "squat": (0, 50, 51), "crouch": True, "seed": n}),
                           ("gyropod", "gyropod", {"seed": n})):
        cfg = _config(kind, **{k: v for k, v in kw.items() if k == "joint_limits"})
        ref = _references(model, oracle_lib, torch, kind, n=n, ticks=ticks, exact=False, **kw)
        dev = _rollout(model, {"device": _Device(torch, model, cfg, n, path)}, kind, n, ticks, seed=n,
                       squat=kw.get("squat"), crouch=kw.get("crouch", False))["device"]
        g, h = _drift(model, dev, ref["oracle"]), _drift(model, ref["host"], ref["oracle"])
        _report(f"tail_lanes_{kind}_{n}", **{f"{k}_{m}": v for k, e in (("device", g), ("host", h)) for m, v in e.items()})
        assert np.array_equal(dev[1], ref["oracle"][1]), (kind, n)
        assert g["pitch"] <= RATIO * h["pitch"] + 2e-7, (kind, n, g, h)
        assert g["pos"] <= RATIO * h["pos"] + 5e-7, (kind, n, g, h)
        assert g["yaw"] <= RATIO * h["yaw"] + 5e-7, (kind, n, g, h)
        assert g["contact"] <= 1, (kind, n, g)
