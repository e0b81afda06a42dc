# SPDX-License-Identifier: Apache-2.0
"""The kernels' per-robot arithmetic (sim_core.cuh / sim_pair.cuh / mpc_core.cuh compiled for the
host, fp32: `HostSim` steps with the same paired-leg substep functions the device runs) against the fp64 oracle. Runs without a GPU; the `-m gpu` tests repeat
the comparisons through the C ABI on the device.

Tolerances (DESIGN.md "Parity"): the fp32 common-frame formulation carries ~1e-5
relative error on accelerations; the Bullet-style contact row has a sensitivity of
1/h = 1000 s^-1 to the penetration depth at touchdown (times 1/r = 20 on wheel
rates), so velocities at touchdown substeps can differ by ~1e-3..1e-2 while
steady contact agrees to ~1e-5.
"""
import numpy as np
import pytest

from conftest import at_joint_bounds, mpc_kkt_residual, random_servo_actions, random_states
from hostsim_wrap import HostSim, mpc_step, philox
from upkie_b200 import _abi


def _pair(model, oracle_lib, n, cfg=None, **kw):
    cfg = cfg if cfg is not None else _abi.default_sim_config()
    for k, v in kw.items():
        setattr(cfg, k, v)
    return HostSim(model, cfg, n), oracle_lib.OracleSim(model, cfg, n, threads=4), cfg


def test_free_flight_substep(model, oracle_lib):
    n = 256
    hs, osim, cfg = _pair(model, oracle_lib, n)
    st = random_states(n, seed=11, z_range=(2.0, 3.0)).astype(np.float32)
    tau = (np.random.default_rng(12).uniform(-1, 1, (n, 6)) * model.tau_max).astype(np.float32)
    hs.set_state(st)
    osim.set_state(st.astype(np.float64))
    for _ in range(5):
        hs.substep(tau)
        osim.substep(tau.astype(np.float64), cfg.dt / cfg.nb_substeps)
    d = np.abs(hs.state[:, :25].astype(np.float64) - osim.get_state()[:, :25])
    assert d[:, :7].max() < 1e-6  # pose
    assert d[:, 13:19].max() < 1e-5  # joint angles
    assert d[:, 7:13].max() < 2e-4 and d[:, 19:25].max() < 2e-3  # velocities (accelerations up to 1e4 rad/s^2)


def test_steady_contact_tick(model, oracle_lib):
    """Robots standing on the ground under a PD action: one 5 ms tick."""
    n = 128
    hs, osim, cfg = _pair(model, oracle_lib, n)
    rng = np.random.default_rng(5)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2] = 0.58
    pitch = rng.uniform(-0.1, 0.1, n)
    init[:, 3], init[:, 5] = np.cos(pitch / 2), np.sin(pitch / 2)
    hs.reset(init)
    osim.reset(init.astype(np.float64))
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, [2, 5], 0] = np.nan
    act[:, :, 3] = act[:, :, 4] = 1.0
    act[:, :, 5] = 0.99 * model.tau_max  # float32(1.7) > 1.7: at the bound itself fp64 clamps, fp32 does not
    act[:, [2, 5], 1] = rng.uniform(-3, 3, (n, 2))
    for _ in range(10):  # settle on the ground
        hs.step_servos(act)
        osim.step_servos(act.astype(np.float64))
    # re-synchronise, then compare one tick
    osim.set_state(hs.state.astype(np.float64))
    gobs, gerr = hs.step_servos(act)
    oobs, _, _, _ = osim.step_servos(act.astype(np.float64))
    d = np.abs(hs.state[:, :25].astype(np.float64) - osim.get_state()[:, :25])
    assert (hs.state[:, 40] == 1).all()
    assert d[:, :7].max() < 1e-6 and d[:, 13:19].max() < 1e-5
    assert d[:, 7:13].max() < 1e-4 and d[:, 19:25].max() < 2e-3
    assert np.abs(gobs[:, :, 2] - oobs[:, :, 2]).max() < 5e-3  # commanded torques
    assert np.array_equal(gerr, osim.error_flags())


def test_random_states_one_tick(model, oracle_lib):
    n = 512
    hs, osim, cfg = _pair(model, oracle_lib, n)
    st = random_states(n, seed=3).astype(np.float32)
    act = random_servo_actions(n, model, seed=4).astype(np.float32)
    hs.set_state(st)
    osim.set_state(st.astype(np.float64))
    gobs, gerr = hs.step_servos(act)
    oobs, orew, oterm, otrunc = osim.step_servos(act.astype(np.float64))
    gs, os_ = hs.state.astype(np.float64), osim.get_state()
    assert np.abs(gs[:, :7] - os_[:, :7]).max() < 2e-5
    assert np.abs(gs[:, 13:19] - os_[:, 13:19]).max() < 2e-4
    dv = np.abs(gs[:, 7:13] - os_[:, 7:13]).max(axis=1)
    dqd = np.abs(gs[:, 19:25] - os_[:, 19:25]).max(axis=1)
    assert np.median(dv) < 5e-5 and np.median(dqd) < 5e-4
    assert dv.max() < 2e-2 and dqd.max() < 0.4  # touchdown outliers, see module docstring
    assert np.array_equal(gs[:, 40], os_[:, 40])  # contact flags bit-exact
    assert np.array_equal(gerr, osim.error_flags())  # clamp / NaN-velocity flags bit-exact
    assert np.array_equal(gobs[:, :, 3:], np.tile(np.array([42.0, 18.0], dtype=np.float32), (n, 6, 1)))
    assert (orew == 0.0).all() and not oterm.any() and not otrunc.any()


def test_fp32_error_budget_against_textbook_fp32(model, oracle_lib):
    """The kernels' fp32 arithmetic stays within a small factor of a textbook link-frame fp32 ABA
    (the oracle instantiated in float) when both are measured against the fp64 oracle. This pins the
    closed-form wheel leaf of legs_pass12 (sim_pair.cuh): taking D = S^T IA S of the wheel about the base
    origin instead loses a factor m |o|^2 / Iyy ~ 150 to cancellation and put the median wheel-rate error
    at 7e-5 rad/s on these inputs (30x the textbook fp32 figure); the closed form brings it to ~1e-5."""
    n = 4096
    cfg = _abi.default_sim_config()
    hs = HostSim(model, cfg, n)
    o64 = oracle_lib.OracleSim(model, cfg, n, threads=4)
    o32 = oracle_lib.OracleSim(model, cfg, n, use_float=True, threads=4)
    st = random_states(n, seed=77).astype(np.float32)
    st[: n // 2, 2] = np.random.default_rng(5).uniform(0.45, 0.62, n // 2)  # half of them on or near the ground
    act = random_servo_actions(n, model, seed=78).astype(np.float32)
    hs.set_state(st)
    o64.set_state(st.astype(np.float64))
    o32.set_state(st.astype(np.float64))
    hp = HostSim(model, cfg, n)  # the paired-leg substep the device runs, reached through the extras entry point
    hp.set_state(st)
    hp.step_servos_ext(act, np.zeros((n, 7, 3), dtype=np.float32))
    hs.step_servos(act)  # the same substep through the plain entry point
    assert np.array_equal(hs.state[:, :25], hp.state[:, :25])
    hsc = HostSim(model, cfg, n, scalar_legs=True)  # the scalar-leg variant (UPKIE_PAIRED_LEGS=0 builds)
    hsc.set_state(st)
    hsc.step_servos(act)
    o64.step_servos(act.astype(np.float64))
    o32.step_servos(act.astype(np.float64))
    ref = o64.get_state()[:, 19:25]
    ep = np.abs(hp.state[:, 19:25].astype(np.float64) - ref).max(axis=1)
    assert np.median(ep) < 2.5e-5, np.median(ep)
    esc = np.abs(hsc.state[:, 19:25].astype(np.float64) - ref).max(axis=1)
    assert np.median(esc) < 2.5e-5, np.median(esc)
    ek = np.abs(hs.state[:, 19:25].astype(np.float64) - ref).max(axis=1)
    et = np.abs(o32.get_state()[:, 19:25] - ref).max(axis=1)
    assert np.median(ek) < 2.5e-5, np.median(ek)
    assert np.median(ek) < 8 * np.median(et)
    assert np.percentile(ek, 99) < 6 * np.percentile(et, 99) + 1e-4
    # wheels (joints 2 and 5) are no worse than the other joints any more
    per_joint = np.median(np.abs(hs.state[:, 19:25].astype(np.float64) - ref), axis=0)
    assert per_joint[[2, 5]].max() < 2.0 * per_joint[[0, 1, 3, 4]].max()


@pytest.mark.parametrize("solver", [1, 2, 3])
def test_joint_limit_rows(model, oracle_lib, solver):
    """btMultiBodyJointLimitConstraint rows against the oracle's restatement, three ticks with a third of the robots
    on a bound, in flight and on the ground. config.joint_limits = 1: the scalar slow path (limit_contact_solve,
    sim_pair.cuh: the limit and contact rows of a robot in one scalar PGS); 2: the packed ten-row solver
    (contact_solve_ten_rows) every robot of the instantiation runs. Two independent implementations, one oracle."""
    n = 2048
    cfg = _abi.default_sim_config()
    cfg.joint_limits = solver
    hs, osim = HostSim(model, cfg, n), oracle_lib.OracleSim(model, cfg, n, threads=4)
    cfg_free = _abi.default_sim_config()
    cfg_free.joint_limits = 0
    free = HostSim(model, cfg_free, n)
    st = at_joint_bounds(model, n, seed=5)
    act = random_servo_actions(n, model, seed=12).astype(np.float32)
    zero = np.zeros((n, 7, 3), dtype=np.float32)
    hs.set_state(st)
    free.set_state(st)
    osim.set_state(st.astype(np.float64))
    lo = np.array([j.limit.lower for j in model.joints])[[0, 1, 3, 4]]
    hi = np.array([j.limit.upper for j in model.joints])[[0, 1, 3, 4]]
    for tick in range(3):
        hs.step_servos_ext(act, zero)  # the paired substep, as the "extras" kernels run it
        free.step_servos_ext(act, zero)
        osim.step_servos(act.astype(np.float64))
        a, b = hs.state.astype(np.float64), osim.get_state()
        d = np.abs(a[:, :25] - b[:, :25])
        assert d[:, :7].max() < 2e-5 and d[:, 13:19].max() < 2e-4
        assert np.median(d[:, 19:25].max(axis=1)) < 5e-5 and np.percentile(d[:, 19:25].max(axis=1), 99) < 2e-3
        assert d[:, 19:25].max() < 0.4  # touchdown outliers as in test_random_states_one_tick
        assert np.array_equal(a[:, 40], b[:, 40])  # contact flags
        q = b[:, 13:19][:, [0, 1, 3, 4]]
        assert ((q < lo) | (q > hi)).any(axis=1).mean() > 0.1  # the rows are exercised on every tick
        assert np.abs(a[:, 19:25] - free.state[:, 19:25]).max() > 5.0  # and they matter
        osim.set_state(hs.state.astype(np.float64))
        free.set_state(hs.state)
    # robots away from their bounds: with the slow path they take the six-row solver (bit-identical with and without
    # the flag), with the ten-row solver their limit slots are empty (same result to round-off)
    st2 = random_states(256, seed=3).astype(np.float32)
    h1, h0 = HostSim(model, cfg, 256), HostSim(model, cfg_free, 256)
    h1.set_state(st2)
    h0.set_state(st2)
    z = np.zeros((256, 7, 3), dtype=np.float32)
    h1.step_servos_ext(act[:256], z)
    h0.step_servos_ext(act[:256], z)
    inside = np.all((st2[:, 13:19][:, [0, 1, 3, 4]] > lo + 0.2) & (st2[:, 13:19][:, [0, 1, 3, 4]] < hi - 0.2), axis=1)
    assert inside.sum() > 100
    if solver == 1:
        assert np.array_equal(h1.state[inside], h0.state[inside])
    else:
        assert np.abs(h1.state[inside][:, :25] - h0.state[inside][:, :25]).max() < 5e-3
        assert np.median(np.abs(h1.state[inside][:, 19:25] - h0.state[inside][:, 19:25])) < 1e-6


def test_joint_limit_stops_a_swinging_knee(model, oracle_lib):
    """What the rows do, on the oracle: a knee swinging at 3 rad/s towards its upper bound in free flight passes
    it by less than 2 mrad and comes back, where without the rows it keeps going."""
    out = {}
    for flag in (0, 1):
        cfg = _abi.default_sim_config()
        cfg.joint_limits = flag
        osim = oracle_lib.OracleSim(model, cfg, 1)
        st = osim.get_state().copy()
        st[0, 2] = 2.0
        st[0, 14], st[0, 20] = 2.45, 3.0
        osim.set_state(st)
        act = np.zeros((1, 6, 6))
        act[:, :, 0] = np.nan
        act[:, :, 5] = 16.0
        traj = []
        for _ in range(40):
            osim.step_servos(act)
            traj.append(osim.get_state()[0, [14, 20]].copy())
        out[flag] = np.array(traj)
    upper = model.joints[1].limit.upper
    assert out[0][-1, 0] > upper + 0.3
    assert out[1][:, 0].max() < upper + 2e-3 and out[1][-1, 1] < 0.0


def test_clamps_match_get_spine_action(model, oracle_lib):
    """UpkieServos.get_spine_action clamps (upkie_servos.py:326-342): values
    outside the box are clamped, NaN positions pass through, flags raised."""
    n = 4
    hs, osim, cfg = _pair(model, oracle_lib, n)
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 5] = 0.99 * model.tau_max
    act[1, 0, 0] = 5.0  # beyond the hip limit 1.26
    act[1, 0, 3] = 9.0  # kp_scale beyond max_gain_scale
    act[2, 2, 2] = 50.0  # feedforward torque beyond 1.7
    act[3, 1, 1] = np.nan  # NaN velocity: asserted in the reference (pybullet_backend.py:519)
    st = random_states(n, seed=1, z_range=(2, 3)).astype(np.float32)
    hs.set_state(st)
    osim.set_state(st.astype(np.float64))
    _, gerr = hs.step_servos(act)
    osim.step_servos(act.astype(np.float64))
    oerr = osim.error_flags()
    # env 3 (NaN velocity) is undefined behaviour in the reference (assertion): the oracle lets the NaN
    # poison the state (np.clip propagates NaN), the kernel's fminf/fmaxf clip drops it; both flag it
    assert np.array_equal(gerr[:3], oerr[:3])
    assert oerr[3] & _abi.ERR_NAN_VELOCITY
    assert gerr[0] == 0
    assert gerr[1] & _abi.ERR_CLAMPED and gerr[2] & _abi.ERR_CLAMPED
    assert gerr[3] & _abi.ERR_NAN_VELOCITY
    # the feedforward torque is clamped to the box, then clipped to maximum_torque (0.99 * 1.7)
    assert hs.state[2, _abi.ST_TORQUE + 2] == np.float32(0.99 * 1.7)


def test_gyropod_and_pendulum_wrappers(model, oracle_lib):
    n = 64
    hs, osim, cfg = _pair(model, oracle_lib, n)
    rng = np.random.default_rng(9)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2] = 0.6
    pitch = rng.uniform(-0.2, 0.2, n)
    init[:, 3], init[:, 5] = np.cos(pitch / 2), np.sin(pitch / 2)
    init[:, 13:19] = rng.uniform(-0.3, 0.3, (n, 6))
    hs.reset(init)
    osim.reset(init.astype(np.float64))
    # UpkieGyropod.reset: leg targets <- observed joint positions, yaw = 0 (upkie_gyropod.py:216-244)
    assert np.allclose(hs.state[:, 34:38], hs.state[:, [13, 14, 16, 17]])
    for t in range(20):
        a = rng.uniform(-4, 4, (n, 2)).astype(np.float32)  # beyond the +-3 / +-1 boxes on purpose
        osim.set_state(hs.state.astype(np.float64))
        g6, gterm = hs.step_gyropod(a, 2)
        o6, orew, oterm, otrunc = osim.step_gyropod(a.astype(np.float64), 2)
        assert np.abs(g6[:, [0, 1, 2, 5]] - o6[:, [0, 1, 2, 5]]).max() < 1e-4
        assert np.median(np.abs(g6[:, 3:5] - o6[:, 3:5])) < 1e-3
        safe = np.abs(np.abs(o6[:, 1]) - cfg.fall_pitch) > 1e-4
        assert np.array_equal(gterm[safe], oterm[safe])
        # yaw integrates the UNCLAMPED action (upkie_gyropod.py:383-385)
        assert np.allclose(g6[:, 5], a[:, 1])
    # pendulum = gyropod with yaw command 0 and obs[[1, 0, 4, 3]] (upkie_pendulum.py:17,137-140)
    a1 = rng.uniform(-3, 3, (n, 1)).astype(np.float32)
    osim.set_state(hs.state.astype(np.float64))
    g6, _ = hs.step_gyropod(a1, 1)
    o4, _, _, _ = osim.step_gyropod(a1.astype(np.float64), 1)
    assert np.abs(g6[:, [1, 0]] - o4[:, [0, 1]]).max() < 1e-4


def test_leg_low_pass_and_wheel_velocity_targets(model, oracle_lib):
    """Closed-form pieces of UpkieGyropod (tests/envs/test_upkie_gyropod.py:56-122):
    pure yaw gives equal-sign wheel velocities, legs low-pass to zero with tau = 1 s."""
    n = 1
    cfg = _abi.default_sim_config()
    cfg.nb_substeps = 1  # the stored torque is then the one computed from the initial (zero) wheel velocities
    hs = HostSim(model, cfg, n)
    st = np.zeros((1, _abi.STATE_DIM), dtype=np.float32)
    st[0, 2], st[0, 3] = 5.0, 1.0
    st[0, 34:38] = [0.4, -0.2, 0.1, 0.3]
    hs.set_state(st)
    hs.step_gyropod(np.array([[0.0, 1.0]], dtype=np.float32), 2)
    alpha = cfg.dt / 1.0
    assert np.allclose(hs.state[0, 34:38], np.array([0.4, -0.2, 0.1, 0.3]) * (1 - alpha), atol=1e-7)
    # in free flight the wheel torques are kd * (target - qd) clipped to 1.7: same sign on both wheels
    tl, tr = hs.state[0, _abi.ST_TORQUE + 2], hs.state[0, _abi.ST_TORQUE + 5]
    assert tl > 0 and tr > 0


def test_inertia_randomization_and_friction(model, oracle_lib):
    n = 64
    hs, osim, cfg = _pair(model, oracle_lib, n)
    rng = np.random.default_rng(2)
    eps = rng.uniform(-0.2, 0.2, (n, 6))
    mu = rng.uniform(0.5, 1.2, n)
    hs.set_randomization(friction=mu, inertia_eps=eps)
    osim.set_randomization(friction=mu.astype(np.float32).astype(np.float64),
                           inertia_eps=eps.astype(np.float32).astype(np.float64))
    st = random_states(n, seed=21).astype(np.float32)
    act = random_servo_actions(n, model, seed=22, torque_mode=True).astype(np.float32)
    hs.set_state(st)
    osim.set_state(st.astype(np.float64))
    hs.step_servos(act)
    osim.step_servos(act.astype(np.float64))
    gs, os_ = hs.state.astype(np.float64), osim.get_state()
    assert np.abs(gs[:, :7] - os_[:, :7]).max() < 2e-5
    assert np.median(np.abs(gs[:, 19:25] - os_[:, 19:25]).max(axis=1)) < 1e-3
    # randomisation changes the dynamics
    hs2 = HostSim(model, cfg, n)
    hs2.set_state(st)
    hs2.step_servos(act)
    assert np.abs(hs2.state[:, 19:25] - hs.state[:, 19:25]).max() > 1e-2


def test_warm_started_contact_impulses(model, oracle_lib):
    """Optional Bullet-style warm start of the normal rows (warmstarting_factor = 0.85): kernel
    arithmetic and oracle agree, the cached impulses are part of the state, and the converged
    contact solution does not depend on the starting point."""
    n = 128
    hs, osim, cfg = _pair(model, oracle_lib, n, warmstarting_factor=0.85)
    hs0, _, _ = _pair(model, oracle_lib, n)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2], init[:, 3] = 0.58, 1.0
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, [2, 5], 0] = np.nan
    act[:, :, 3] = act[:, :, 4] = 1.0
    act[:, :, 5] = 0.99 * model.tau_max
    act[:, [2, 5], 1] = np.random.default_rng(0).uniform(-3, 3, (n, 2))
    for sim in (hs, osim, hs0):
        sim.reset(init if sim is not osim else init.astype(np.float64))
    for _ in range(10):
        hs.step_servos(act)
        hs0.step_servos(act)
        osim.step_servos(act.astype(np.float64))
    lam = hs.state[:, _abi.ST_CONTACT_IMPULSE:_abi.ST_CONTACT_IMPULSE + 2]
    weight_impulse = 5.3382 * 9.81 * cfg.dt / cfg.nb_substeps / 2  # half the weight per wheel over one substep
    assert np.abs(lam - weight_impulse).max() < 0.3 * weight_impulse
    assert np.abs(lam - osim.get_state()[:, _abi.ST_CONTACT_IMPULSE:_abi.ST_CONTACT_IMPULSE + 2]).max() < 1e-4
    d = np.abs(hs.state[:, :25].astype(np.float64) - osim.get_state()[:, :25])
    assert d[:, :7].max() < 1e-5 and d[:, 19:25].max() < 5e-3
    assert np.abs(hs.state[:, :25] - hs0.state[:, :25]).max() < 5e-3  # cold and warm start: same fixed point


def test_spine_observation(model, oracle_lib):
    n = 128
    hs, osim, cfg = _pair(model, oracle_lib, n)
    st = random_states(n, seed=7).astype(np.float32)
    act = random_servo_actions(n, model, seed=8).astype(np.float32)
    hs.set_state(st)
    osim.set_state(st.astype(np.float64))
    hs.step_servos(act)
    osim.step_servos(act.astype(np.float64))
    g, o = hs.spine_obs().astype(np.float64), osim.spine_obs()
    assert np.abs(g[:, 16:20] - o[:, 16:20]).max() < 1e-4  # IMU quaternion incl. scipy's sign convention
    assert np.abs(g[:, 6] - o[:, 6]).max() < 1e-5  # pitch
    assert np.abs(g[:, 7:16] - o[:, 7:16]).max() < 1e-5
    assert np.array_equal(g[:, 29], o[:, 29])
    assert np.abs(g[:, 60] - o[:, 60]).max() < 1e-5
    assert np.array_equal(g[:, 30:60].reshape(n, 6, 5)[:, :, 3:], o[:, 30:60].reshape(n, 6, 5)[:, :, 3:])


def test_twenty_tick_trajectory_under_pd(model, oracle_lib):
    """Short closed-loop horizon without re-synchronisation (README PD policy,
    README.md:62-64): fp32 and fp64 trajectories stay close for 0.1 s."""
    n = 32
    hs, osim, cfg = _pair(model, oracle_lib, n)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2], init[:, 3] = 0.6, 1.0
    hs.reset(init)
    osim.reset(init.astype(np.float64))
    go, oo = np.zeros((n, 6)), np.zeros((n, 4))
    for t in range(20):
        ga = (10.0 * go[:, 1] + 1.0 * go[:, 0] + 0.0 * go[:, 4] + 0.1 * go[:, 3]).reshape(n, 1)
        oa = (10.0 * oo[:, 0] + 1.0 * oo[:, 1] + 0.0 * oo[:, 2] + 0.1 * oo[:, 3]).reshape(n, 1)
        g6, gterm = hs.step_gyropod(ga.astype(np.float32), 1)
        oo, _, oterm, _ = osim.step_gyropod(oa, 1)
        go = g6.astype(np.float64)
    assert np.abs(go[:, 1] - oo[:, 0]).max() < 1e-3  # pitch
    assert np.abs(go[:, 0] - oo[:, 1]).max() < 1e-3  # ground position
    assert np.array_equal(gterm, oterm)


def test_two_second_closed_loop_stays_on_the_oracle(model, oracle_lib):
    """400 ticks (2 s) of the README PD policy from initial pitches in +-0.25 rad, each side closing the loop on its
    OWN observations, no re-synchronisation: the fp32 kernel arithmetic stays within 1e-4 rad / 5e-4 m of the fp64
    oracle for every robot, and `terminated` agrees on every tick (measured: 4e-6 rad, 5e-5 m over 1 024 robots)."""
    n, ticks = 256, 400
    hs, osim, cfg = _pair(model, oracle_lib, n)
    pitch = np.random.default_rng(0).uniform(-0.25, 0.25, n)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2], init[:, 3], init[:, 5] = 0.6, np.cos(pitch / 2), np.sin(pitch / 2)
    hs.reset(init)
    osim.reset(init.astype(np.float64))
    go, oo = np.zeros((n, 6)), np.zeros((n, 4))
    for t in range(ticks):
        ga = (10.0 * go[:, 1] + 1.0 * go[:, 0] + 0.1 * go[:, 3]).reshape(n, 1)
        oa = (10.0 * oo[:, 0] + 1.0 * oo[:, 1] + 0.1 * oo[:, 3]).reshape(n, 1)
        g6, gterm = hs.step_gyropod(ga.astype(np.float32), 1)
        oo, _, oterm, _ = osim.step_gyropod(oa, 1)
        go = g6.astype(np.float64)
        assert np.array_equal(gterm, oterm), t
        if t % 50 == 49:
            assert np.abs(go[:, 1] - oo[:, 0]).max() < 1e-4, t  # pitch
            assert np.abs(go[:, 0] - oo[:, 1]).max() < 5e-4, t  # ground position
    assert np.abs(oo[:, 0]).max() < 0.5  # nobody fell: the comparison above is about balancing robots


def test_wheel_contact_points_follow_the_collision_pass(model, oracle_lib):
    """Host-side contact query of the Backend adapter (``PyBulletBackend.get_contact_points``): a contact point is
    reported exactly when the oracle's collision pass saw one, it lies on the tire under the wheel centre, and for
    a robot at rest the two normal forces carry its weight."""
    from upkie_b200.model import wheel_contact_points

    n = 512
    cfg = _abi.default_sim_config()
    osim = oracle_lib.OracleSim(model, cfg, n, threads=4)
    st = random_states(n, seed=21)
    st[:, 7:13] *= 0.05  # slow base motion: the contact flag of the last substep then describes the final pose
    st[:, 19:25] *= 0.05
    osim.set_state(st.astype(np.float64))
    act = np.zeros((n, 6, 6))
    act[:, :, 0] = np.nan
    act[:, :, 5] = 1.0
    osim.step_servos(act)
    rows = osim.get_state()
    h = cfg.dt / cfg.nb_substeps
    agree = 0
    for i in range(n):
        pts = wheel_contact_points(model, rows[i], h)
        # the flag belongs to the collision pass at the START of the last substep: skip robots within 2 mm of the
        # threshold at the end of it
        near = [abs(p[2] - 0.02) < 2e-3 for _, p, _ in wheel_contact_points(model, rows[i], h, breaking_threshold=1e9)]
        if any(near):
            continue
        assert (len(pts) > 0) == (rows[i, _abi.ST_CONTACT] > 0.5), i
        agree += 1
        for side, p, force in pts:
            assert p[2] < 0.02 and force[2] >= 0.0
    assert agree > 0.9 * n
    # a robot standing still on its wheels
    osim1 = oracle_lib.OracleSim(model, cfg, 1)
    init = np.zeros((1, _abi.INIT_DIM))
    init[:, 2], init[:, 3] = 0.6, 1.0
    osim1.reset(init)
    hold = np.zeros((1, 6, 6))
    hold[:, :, 3], hold[:, :, 4], hold[:, :, 5] = 1.0, 1.0, np.asarray(model.tau_max)
    for _ in range(40):
        osim1.step_servos(hold)
    pts = wheel_contact_points(model, osim1.get_state()[0], h)
    assert [s for s, _, _ in pts] == [0, 1]
    total = sum(f[2] for _, _, f in pts)
    assert abs(total - float(np.sum(model.mass)) * cfg.gravity) < 0.15 * float(np.sum(model.mass)) * cfg.gravity
    assert all(np.linalg.norm(f[:2]) < 0.05 * f[2] for _, _, f in pts)  # at rest on flat ground: hardly any friction
    (_, pl, _), (_, pr, _) = pts
    assert abs(pl[2]) < 5e-3 and abs(pr[2]) < 5e-3 and abs((pl[1] - pr[1]) - model.wheel_base) < 1e-3
    from upkie_b200.model import contact_points_from_state

    row = osim1.get_state()[0]
    contacts = contact_points_from_state(model, row, cfg)
    assert [c.link_name for c in contacts] == ["left_wheel_tire", "right_wheel_tire"]
    assert np.allclose(contacts[0].force_in_world, pts[0][2])
    assert [c.link_name for c in contact_points_from_state(model, row, cfg, "right_wheel_tire")] == ["right_wheel_tire"]
    assert contact_points_from_state(model, row, cfg, "imu") == [] == contact_points_from_state(model, row, cfg, "nope")
    assert "PointContact(link_name='left_wheel_tire'" in repr(contacts[0])


def test_contact_points_report_the_friction_force(model, oracle_lib):
    """``get_contact_points`` sums normal force and the two friction components (pybullet_backend.py:696-709). A robot
    held upright by its servos and pushed sideways with 10 N (below mu W = 52 N) stays put: the tires' friction forces
    balance the push, the normal forces the weight - for the oracle and for the kernels' arithmetic."""
    from upkie_b200.model import contact_points_from_state

    cfg = _abi.default_sim_config()
    push = np.zeros((1, 7, 3))
    push[0, 0] = [0.0, 10.0, 0.0]  # newtons on the base, world frame
    hold = np.zeros((1, 6, 6))
    hold[:, :, 3], hold[:, :, 4], hold[:, :, 5] = 1.0, 1.0, np.asarray(model.tau_max)
    init = np.zeros((1, _abi.INIT_DIM))
    init[:, 2], init[:, 3] = 0.6, 1.0
    osim = oracle_lib.OracleSim(model, cfg, 1)
    osim.reset(init)
    hs = HostSim(model, cfg, 1)
    hs.reset(init.astype(np.float32))
    osim.set_external_forces(push)
    for _ in range(60):
        osim.step_servos(hold)
        hs.step_servos_ext(hold.astype(np.float32), push.astype(np.float32))
    weight = float(np.sum(model.mass)) * cfg.gravity
    for row in (osim.get_state()[0], hs.state[0]):
        contacts = contact_points_from_state(model, row, cfg)
        assert len(contacts) == 2
        total = sum(c.force_in_world for c in contacts)
        assert abs(total[1] + 10.0) < 1.5, total   # friction balances the push
        assert abs(total[2] - weight) < 0.15 * weight
        assert abs(total[0]) < 2.0
        assert abs(row[8]) < 5e-3  # and the robot does not slide (base y velocity)


def test_imu_uncertainty_known_answers(model):
    """ImuUncertainty on the spine observation (`apply_imu_uncertainty`, as `k_spine_obs` calls it) against the
    reference's own cases (upkie/cpp/interfaces/tests/ImuUncertaintyTest.cpp:23-41): no bias and no noise leaves the
    observation alone; a pure bias is added exactly, to the filtered and raw accelerations and the angular velocity,
    and to nothing else; white noise has the configured standard deviation and independent raw / filtered draws."""
    n = 4096
    st = random_states(n, seed=41).astype(np.float32)

    def spine(cfg, tick=7):
        hs = HostSim(model, cfg, n)
        hs.set_state(st)
        return hs.spine_obs(), hs.spine_obs_with_uncertainty(tick)

    plain, same = spine(_abi.default_sim_config())
    assert np.array_equal(plain, same)  # NoBiasNoNoise
    cfg = _abi.default_sim_config()
    acc_bias, gyro_bias = (0.1, -0.2, 0.3), (-0.01, 0.02, 0.03)
    for k in range(3):
        cfg.imu_accelerometer_bias[k], cfg.imu_gyroscope_bias[k] = acc_bias[k], gyro_bias[k]
    plain, biased = spine(cfg)
    d = biased.astype(np.float64) - plain
    s_acc, s_raw, s_gyr = _abi.SP_IMU_LINACC, _abi.SP_IMU_RAWACC, _abi.SP_IMU_ANGVEL
    assert np.abs(d[:, s_acc:s_acc + 3] - acc_bias).max() < 2e-6  # PureBias (fp32 round-off of the sum)
    assert np.abs(d[:, s_raw:s_raw + 3] - acc_bias).max() < 2e-6
    assert np.abs(d[:, s_gyr:s_gyr + 3] - gyro_bias).max() < 2e-6
    other = np.ones(_abi.SPINE_DIM, dtype=bool)
    for s0 in (s_acc, s_raw, s_gyr):
        other[s0:s0 + 3] = False
    assert np.array_equal(biased[:, other], plain[:, other])
    cfg = _abi.default_sim_config()
    cfg.imu_accelerometer_noise, cfg.imu_gyroscope_noise, cfg.noise_seed = 0.5, 0.05, 3
    plain, noisy = spine(cfg)
    d = noisy.astype(np.float64) - plain
    assert abs(d[:, s_acc:s_acc + 3].std() / 0.5 - 1) < 0.03 and abs(d[:, s_gyr:s_gyr + 3].std() / 0.05 - 1) < 0.03
    assert abs(d[:, s_raw:s_raw + 3].std() / 0.5 - 1) < 0.03 and abs(d[:, s_acc:s_acc + 3].mean()) < 0.02
    assert abs(np.corrcoef(d[:, s_acc], d[:, s_raw])[0, 1]) < 0.05  # raw and filtered: independent draws
    _, again = spine(cfg)
    assert np.array_equal(again, noisy)  # counter-based: repeatable
    _, later = spine(cfg, tick=8)
    assert not np.array_equal(later[:, s_acc], noisy[:, s_acc])


# ---- counter-based RNG ------------------------------------------------------------------------

def test_philox4x32_10_known_answers():
    """Random123 known-answer vectors of Philox4x32-10 (kat_vectors: counter words, key words, output)."""
    kats = [
        ((0, 0, 0, 0), (0, 0), (0x6627E8D5, 0xE169C58D, 0xBC57AC4C, 0x9B00DBD8)),
        ((0xFFFFFFFF,) * 4, (0xFFFFFFFF,) * 2, (0x408F276D, 0x41C83B0E, 0xA20BC7C6, 0x6D5451FD)),
        ((0x243F6A88, 0x85A308D3, 0x13198A2E, 0x03707344), (0xA4093822, 0x299F31D0),
         (0xD16CFE09, 0x94FDCCEB, 0x5001E420, 0x24126EA1)),
    ]
    for c, k, expect in kats:
        assert philox(c[0] | (c[1] << 32), c[2] | (c[3] << 32), k[0] | (k[1] << 32)) == list(expect)


def test_device_sampler_statistics_and_determinism(model):
    cfg = _abi.default_sim_config()
    cfg.rand_pitch, cfg.rand_roll, cfg.rand_x, cfg.rand_z = 0.3, 0.1, 0.05, 0.1
    cfg.rand_omega_x, cfg.rand_omega_y = 0.2, 0.5
    cfg.rand_linear_velocity[0], cfg.rand_linear_velocity[2] = 0.3, 0.1
    n = 4096
    hs = HostSim(model, cfg, n)
    a = hs.sample_init(seed=7, env_offset=0, episode=1)
    b = hs.sample_init(seed=7, env_offset=0, episode=1)
    assert np.array_equal(a, b)
    # sharding invariance: env i of a shard with offset k equals env k + i of the full batch
    hs2 = HostSim(model, cfg, 128)
    c = hs2.sample_init(seed=7, env_offset=1000, episode=1)
    assert np.array_equal(c, a[1000:1128])
    assert not np.array_equal(hs.sample_init(seed=7, env_offset=0, episode=2), a)
    assert np.abs(a[:, 0]).max() <= 0.05 and a[:, 2].min() >= 0.6 and a[:, 2].max() <= 0.7
    pitch = 2 * np.arctan2(a[:, 5], a[:, 3])
    assert np.abs(pitch).max() <= 0.3 + 0.11 and abs(pitch.mean()) < 0.02 and pitch.std() > 0.1
    assert np.abs(a[:, 10]).max() <= 0.2 and np.abs(a[:, 11]).max() <= 0.5 and (a[:, 12] == 0).all()
    assert np.allclose(np.linalg.norm(a[:, 3:7], axis=1), 1.0, atol=1e-6)


def test_device_sampler_draws_around_the_nominal_state(model):
    """Round-1 advisor finding: the on-device sampler of the fused auto-reset ignored the nominal joint configuration
    and base velocities of the initial state. RobotState.sample_state keeps ``joint_configuration`` and ADDS the
    random velocity parts to the nominal ones (upkie/utils/robot_state.py:175-196); so must auto-reset episodes."""
    from upkie_b200.robot_state import RobotState, RobotStateRandomization

    crouch = np.array([0.4, -0.8, 0.0, -0.4, 0.8, 0.0])
    nominal = RobotState(
        joint_configuration=crouch, position_base_in_world=np.array([0.1, 0.0, 0.5]),
        angular_velocity_base_in_base=np.array([0.0, 0.3, 0.1]),
        linear_velocity_base_to_world_in_world=np.array([0.5, 0.0, -0.2]),
        randomization=RobotStateRandomization(pitch=0.2, omega_y=0.4, linear_velocity=np.array([0.3, 0.0, 0.0])),
    )
    cfg = _abi.default_sim_config()
    nominal.apply_to_config(cfg)
    n = 2048
    a = HostSim(model, cfg, n).sample_init(seed=11, env_offset=0, episode=3)
    assert np.allclose(a[:, _abi.INIT_Q:_abi.INIT_Q + 6], crouch.astype(np.float32))
    assert (a[:, _abi.INIT_QD:_abi.INIT_QD + 6] == 0).all()
    om, v = a[:, _abi.INIT_ANGVEL:_abi.INIT_ANGVEL + 3], a[:, _abi.INIT_LINVEL:_abi.INIT_LINVEL + 3]
    assert np.allclose(om[:, 0], 0.0) and np.allclose(om[:, 2], 0.1) and np.abs(om[:, 1] - 0.3).max() <= 0.4 + 1e-6
    assert om[:, 1].std() > 0.15 and abs(om[:, 1].mean() - 0.3) < 0.03
    assert np.abs(v[:, 0] - 0.5).max() <= 0.3 + 1e-6 and np.allclose(v[:, 2], -0.2) and v[:, 0].std() > 0.1
    assert np.allclose(a[:, 0], 0.1) and np.allclose(a[:, 2], 0.5)
    # the same bounds through the reference-order host sampler: same ranges, same nominal values
    rows = np.stack([nominal.sample_state(np.random.default_rng(s)).to_row() for s in range(256)])
    assert np.allclose(rows[:, _abi.INIT_Q:_abi.INIT_Q + 6], crouch)
    assert abs(rows[:, _abi.INIT_ANGVEL + 1].mean() - 0.3) < 0.08 and np.allclose(rows[:, _abi.INIT_ANGVEL + 2], 0.1)
    assert abs(rows[:, _abi.INIT_LINVEL].mean() - 0.5) < 0.06


# ---- MPC ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("horizon", [16, 50])
def test_mpc_riccati_active_set_matches_condensed_oracle(oracle_lib, horizon):
    cfg = _abi.default_mpc_config()
    cfg.nb_timesteps = horizon
    om = oracle_lib.OracleMpc(cfg)
    rng = np.random.default_rng(0)
    n = 300
    x0 = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.2, 0.2, n), rng.uniform(-0.5, 0.5, n),
                   rng.uniform(-1, 1, n)], 1)
    x0[:20, 1] = rng.uniform(0.3, 0.9, 20)  # large pitch: many saturated inputs
    x0[20:30, 1] = rng.uniform(1.05, 1.3, 10)  # fallen
    vt = rng.uniform(-1, 1, n)
    contact = np.ones(n, dtype=np.uint8)
    contact[30:40] = 0
    v0 = rng.uniform(-1, 1, n)
    vc_o, first_o, found_o, plan_o = om.step(x0, vt, contact, 0.005, v0)
    assert found_o.all()
    # same formulation in fp64: agreement to round-off (two independent formulations, one optimum)
    vc64, plan64, found64, it64 = mpc_step(cfg, x0, vt, contact, 0.005, v0, double=True)
    assert found64.all() and np.abs(plan64 - plan_o).max() < 1e-8
    # what the kernel runs (fp32): ProxQP's own tolerance is eps_abs = 1e-3 (mpc_balancer.py:76)
    vc32, plan32, found32, it32 = mpc_step(cfg, x0, vt, contact, 0.005, v0, double=False)
    assert found32.all()
    assert np.abs(plan32[:, 0] - plan_o[:, 0]).max() < 1e-3
    # accuracy gate of config 4 (SURVEY.md 8d): KKT residual of the fp32 plan in the fp64 condensed QP <= 1e-3
    om = oracle_lib.OracleMpc(cfg)
    Pm, _, _ = om.matrices()
    live = np.flatnonzero((np.abs(x0[:, 1]) <= 1.0) & (contact != 0))[:96]
    worst = max(mpc_kkt_residual(Pm, om.cost_vector(x0[i].astype(np.float64), float(vt[i])), plan32[i], cfg.max_ground_accel)
                for i in live)
    assert worst < 1e-3, worst
    assert np.abs(plan32 - plan_o).max() < 5e-3
    assert np.abs(vc32 - vc_o).max() < 1e-5
    assert it32.max() <= 12
    # MPCBalancer.step post-processing (mpc_balancer.py:295-311)
    fallen = np.abs(x0[:, 1]) > 1.0
    lp = fallen | (contact == 0)
    assert np.allclose(vc_o[lp], v0[lp] * (1 - 0.005 / 0.1))
    ok = ~lp
    assert np.allclose(vc_o[ok], np.clip(v0[ok] + plan_o[ok, 0] * 0.005 / 2.0, -3, 3))
    assert (np.abs(plan_o).max(axis=1) >= 10.0 - 1e-9).sum() >= 20  # saturated cases are exercised


def test_mpc_oracle_against_scipy_bvls(oracle_lib):
    """The oracle's QP solver against an independent bounded least-squares solver."""
    from scipy.optimize import lsq_linear

    cfg = _abi.default_mpc_config()
    om = oracle_lib.OracleMpc(cfg)
    P, A, B = om.matrices()
    L = np.linalg.cholesky(P)
    rng = np.random.default_rng(3)
    for _ in range(8):
        x0 = np.array([rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(-0.5, 0.5), rng.uniform(-1, 1)])
        q = om.cost_vector(x0, rng.uniform(-1, 1))
        U, ok = om.solve(q)
        r = lsq_linear(L.T, -np.linalg.solve(L, q), bounds=(-10, 10), method="bvls", tol=1e-14)
        assert ok and np.abs(U - r.x).max() < 1e-8


def test_mpc_model_matrices(oracle_lib):
    """qpmpc WheeledInvertedPendulum discretisation: A, B satisfy theta'' = w^2 theta - u / l
    and p'' = u (SURVEY.md 8c)."""
    cfg = _abi.default_mpc_config()
    om = oracle_lib.OracleMpc(cfg)
    P, A, B = om.matrices()
    T, g, l = cfg.sampling_period, cfg.gravity, cfg.leg_length
    w = np.sqrt(g / l)
    assert np.allclose(A[0], [1, 0, T, 0]) and np.allclose(A[2], [0, 0, 1, 0])
    assert A[1, 1] == pytest.approx(np.cosh(T * w)) and A[3, 1] == pytest.approx(w * np.sinh(T * w))
    assert np.allclose(B, [T * T / 2, (1 - np.cosh(T * w)) / g, T, -w * np.sinh(T * w) / g])
    # zero-order-hold consistency against a fine explicit integration of the ODE
    x = np.array([0.1, 0.05, -0.2, 0.3])
    u = 2.0
    y = x.copy()
    m = 20000
    for _ in range(m):
        h = T / m
        y = y + h * np.array([y[2], y[3], u, w * w * y[1] - u / l])
    assert np.allclose(A @ x + B * u, y, atol=1e-5)
    assert np.allclose(P, P.T) and np.linalg.eigvalsh(P).min() > 0


def test_gaussian_noise_generator():
    """Philox + Box-Muller normals of the torque noise models: moments, independence, determinism."""
    from hostsim_wrap import gaussian8

    x = np.stack([gaussian8(7, env, tick, slot) for env in range(40) for tick in range(1, 26) for slot in (0, 4, 255)])
    assert x.shape == (3000, 8) and np.isfinite(x).all()
    assert abs(x.mean()) < 0.02 and abs(x.std() - 1.0) < 0.02
    assert abs(((x - x.mean()) ** 4).mean() / x.var() ** 2 - 3.0) < 0.15  # Gaussian kurtosis
    c = np.corrcoef(x.T)
    assert np.abs(c - np.eye(8)).max() < 0.08  # the 8 lanes are independent
    assert np.array_equal(gaussian8(7, 3, 9, 2), gaussian8(7, 3, 9, 2))
    for other in (gaussian8(8, 3, 9, 2), gaussian8(7, 4, 9, 2), gaussian8(7, 3, 10, 2), gaussian8(7, 3, 9, 3)):
        assert not np.array_equal(gaussian8(7, 3, 9, 2), other)


def test_torque_noise_models(model):
    """JointProperties noise (pybullet_backend.py:457-466,545-552): control noise enters before the clip and
    is redrawn every substep, measurement noise only touches the observed torque, sigma <= 1e-10 means off."""
    n = 4000
    cfg = _abi.default_sim_config()
    sig_c = [0.05, 0.0, 0.02, 0.05, 0.0, 0.02]
    sig_m = [0.0, 0.03, 0.01, 0.0, 0.03, 0.01]
    for j in range(6):
        cfg.torque_control_noise[j] = sig_c[j]
        cfg.torque_measurement_noise[j] = sig_m[j]
    cfg.noise_seed = 99
    hs = HostSim(model, cfg, n)
    st = random_states(n, seed=3, z_range=(2.0, 3.0)).astype(np.float32)
    hs.set_state(st)
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 2] = 0.5 * model.tau_max  # pure feedforward torque, kp = kd = 0
    act[:, :, 5] = model.tau_max
    obs = hs.step_servos_noise(act, tick=1)
    applied = hs.state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6]  # torque of the last substep
    ff = 0.5 * np.asarray(model.tau_max, dtype=np.float32)
    for j in range(6):
        d = applied[:, j] - ff[j]
        if sig_c[j] == 0.0:
            assert np.array_equal(applied[:, j], np.full(n, ff[j], dtype=np.float32))
        else:
            assert abs(d.mean()) < 4 * sig_c[j] / np.sqrt(n) and abs(d.std() / sig_c[j] - 1) < 0.05
        m = obs[:, j, 2] - applied[:, j]
        if sig_m[j] == 0.0:
            assert np.array_equal(obs[:, j, 2], applied[:, j])
        else:
            assert abs(m.mean()) < 4 * sig_m[j] / np.sqrt(n) and abs(m.std() / sig_m[j] - 1) < 0.05
    # noise of successive ticks is independent, and the same (seed, env, tick) reproduces it
    first = applied.copy()
    hs.step_servos_noise(act, tick=2)
    second = hs.state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6].copy()
    assert abs(np.corrcoef(first[:, 0] - ff[0], second[:, 0] - ff[0])[0, 1]) < 0.06
    hs.set_state(st)
    hs.step_servos_noise(act, tick=1)
    assert np.array_equal(hs.state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6], first)
    # control noise is clipped with the rest of the command
    act[:, :, 2] = model.tau_max
    act[:, :, 5] = 0.9 * np.asarray(model.tau_max, dtype=np.float32)
    hs.set_state(st)
    hs.step_servos_noise(act, tick=3)
    lim = 0.9 * np.asarray(model.tau_max, dtype=np.float32)
    assert (np.abs(hs.state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6]) <= lim + 1e-6).all()


@pytest.mark.parametrize("local_mask", [0, 0x7F, 0b0101010])
def test_external_forces_match_oracle(model, oracle_lib, local_mask):
    """set_external_forces (pybullet_backend.py:603-658): the kernel applies a force on body i as J_i^T w
    (ancestor joint torques + base wrench); the oracle puts it into the ABA bias force of the body itself."""
    n = 256
    hs, osim, cfg = _pair(model, oracle_lib, n)
    rng = np.random.default_rng(21)
    st = random_states(n, seed=22, z_range=(2.0, 3.0)).astype(np.float32)  # free flight: no contact sensitivity
    ext = rng.uniform(-20.0, 20.0, (n, 7, 3)).astype(np.float32)
    ext[: n // 4, 1:] = 0.0  # base-only pushes
    ext[n // 4: n // 2, 0] = 0.0
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 2] = rng.uniform(-0.5, 0.5, (n, 6)) * model.tau_max
    act[:, :, 5] = 0.99 * np.asarray(model.tau_max, dtype=np.float32)
    hs.set_state(st)
    osim.set_state(st.astype(np.float64))
    osim.set_external_forces(ext.astype(np.float64), local_mask)
    hs.step_servos_ext(act, ext, local_mask)
    osim.step_servos(act.astype(np.float64))
    d = np.abs(hs.state[:, :25].astype(np.float64) - osim.get_state()[:, :25])
    assert d[:, :7].max() < 2e-6 and d[:, 13:19].max() < 2e-5
    assert d[:, 7:13].max() < 3e-4 and d[:, 19:25].max() < 4e-3
    # and the forces do something: same tick without them differs
    hs2 = HostSim(model, cfg, n)
    hs2.set_state(st)
    hs2.step_servos(act)
    assert np.abs(hs2.state[:, 7:10] - hs.state[:, 7:10]).max() > 1e-3
    # physics check of the oracle itself: from rest, one substep changes the total linear momentum by
    # (sum of external forces + weight) * h, wherever the forces act
    if local_mask == 0:
        mass = float(np.sum(model.mass))
        o2 = oracle_lib.OracleSim(model, cfg, 4, threads=1)
        s4 = random_states(4, seed=5, z_range=(2.0, 3.0))
        s4[:, 7:13] = 0.0
        s4[:, 19:25] = 0.0
        o2.set_state(s4)
        f4 = rng.uniform(-20.0, 20.0, (4, 7, 3))
        o2.set_external_forces(f4, 0)
        o2.substep(np.zeros((4, 6)), 1e-5)
        for i in range(4):
            expect = (f4[i].sum(axis=0) + np.array([0.0, 0.0, -mass * cfg.gravity])) * 1e-5
            # O(h^2) slack: the momentum is read after the position update
            assert np.allclose(o2.energy(i)["linear_momentum"], expect, atol=1e-8, rtol=1e-4)


def test_frozen_lanes_keep_bullets_result(model, oracle_lib):
    """Bullet's residual exit rule per lane (DESIGN.md section 3): a robot whose sweep met the threshold is frozen while
    the rest of its warp finishes. With the warp vote forced to "somebody is still sweeping" the robot stays in the loop
    for all 50 trips - its state must come out bit for bit as when it leaves on its own, for the six-row, the ten-row
    and the scalar solvers; and with the threshold at 0 nobody leaves early."""
    import hostsim_wrap

    n = 96
    st = random_states(n, seed=21).astype(np.float32)
    st[:48] = at_joint_bounds(model, 48, seed=22)  # robots on a hip / knee bound: the ten-row solver
    act = random_servo_actions(n, model, seed=23).astype(np.float32)
    results = {}
    for limits in (3, 1, 0):
        for vote in (0, 1):
            cfg = _abi.default_sim_config()
            cfg.joint_limits = limits
            hs = HostSim(model, cfg, n)
            hs.set_state(st)
            hostsim_wrap.lib().hostsim_set_vote_always(vote)
            try:
                for _ in range(3):
                    hs.step_servos(act)
            finally:
                hostsim_wrap.lib().hostsim_set_vote_always(0)
            results[(limits, vote)] = hs.state.copy()
        np.testing.assert_array_equal(results[(limits, 0)], results[(limits, 1)])
    # the threshold matters: all 50 sweeps give (slightly) different impulses, and still match the oracle run the same way
    cfg0 = _abi.default_sim_config()
    cfg0.solver_residual_threshold = 0.0
    hs0, osim0 = HostSim(model, cfg0, n), oracle_lib.OracleSim(model, cfg0, n, threads=4)
    hs0.set_state(st)
    osim0.set_state(st.astype(np.float64))
    hs0.step_servos(act)
    osim0.step_servos(act.astype(np.float64))
    assert np.abs(hs0.state[:, 19:25] - results[(3, 0)][:, 19:25]).max() > 0  # not the same iteration count
    d = np.abs(hs0.state[:, :25].astype(np.float64) - osim0.get_state()[:, :25])
    assert np.median(d[:, 19:25].max(axis=1)) < 5e-4


def test_config_keeps_the_substep_rotation_in_the_integrators_range(model):
    """The base-orientation integrator evaluates polynomials of sin(x) / x and cos(x), fp32-exact for x = |w| h / 2 up
    to 0.52: a config whose substep h and velocity clamp allow more is refused when the parameters are built."""
    import ctypes as C

    import hostsim_wrap

    L, m = hostsim_wrap.lib(), model.to_struct()
    for dt, nb, vmax, ok in ((0.005, 5, 100.0, True), (0.005, 1, 100.0, True), (0.02, 1, 100.0, False),
                             (0.005, 1, 150.0, False), (0.02, 1, 25.0, True)):
        cfg = _abi.default_sim_config()
        cfg.dt, cfg.nb_substeps, cfg.max_coordinate_velocity = dt, nb, vmax
        h = L.hostsim_create(C.byref(m), C.byref(cfg))
        assert bool(h) == ok, (dt, nb, vmax)
        if h:
            L.hostsim_destroy(h)


def _config_cases():
    """One (row, path) of test_gpu_config_parity.VARIANTS per distinct physics: on the host the headline and table
    paths compute what limits3 does."""
    from test_gpu_config_parity import CASES, PATHS

    seen, out = set(), []
    for row, path in CASES:
        if (row,) + PATHS[path][:3] not in seen:
            seen.add((row,) + PATHS[path][:3])
            out.append((row, path))
    return out


HOST_RATIO = 10.0  # measured: the host build's error is 0.5x to 8x the fp32 oracle's on these rows (8x: spine, 100 Hz)


@pytest.mark.parametrize("row,path", _config_cases())
def test_host_build_away_from_the_default_config(model, oracle_lib, row, path):
    """The CPU twin of test_gpu_config_parity.py: one tick of the same robots under each row's configuration, the host
    build against the fp64 oracle. The row bites (it moves the fp64 one-tick state by BITE x the fp32 sides' 99th
    percentile error) and its inputs reach the code under test (body contact rows, spine-mode contact), the host
    build's base twist, joint rates and impulses stay within HOST_RATIO x the fp32 oracle's
    error plus the GPU test's floors, worst robot and 99th percentile, and it flips at most one contact flag more."""
    import test_gpu_config_parity as G

    refs = G.references(model, oracle_lib, row, path)
    ref = refs["oracle"]
    flips = {k: G.contact_mismatch(refs[k], ref) for k in ("oracle32", "host")}
    assert flips["host"].sum() <= flips["oracle32"].sum() + 1
    mask = ~(flips["oracle32"] | flips["host"])
    err = {k: G.errors(refs[k], ref, mask) for k in ("oracle32", "host")}
    move, fp32 = G.bite(refs)
    assert move >= G.BITE * fp32, (row, path, move, fp32)
    G.check_inputs_exercise_the_path(refs, path)
    for g in G.GROUPS:
        for i, q in enumerate(("worst", "p99")):
            assert err["host"][g][i] <= HOST_RATIO * err["oracle32"][g][i] + G.FLOOR[g], (row, path, g, q, err)


def test_friction_rows_sit_on_their_bounds_at_friction_0_1(model, oracle_lib):
    """The friction_0.1 row of test_gpu_config_parity.py binds: on the fp64 oracle, a friction impulse of more than a
    hundred wheels is at +-mu times the wheel's normal impulse."""
    import test_gpu_config_parity as G

    st = G.references(model, oracle_lib, "friction_0.1", "limits3")["oracle"][0]
    lam_n = np.repeat(st[:, _abi.ST_CONTACT_IMPULSE:_abi.ST_CONTACT_IMPULSE + 2], 2, axis=1)
    lam_t = np.abs(st[:, _abi.ST_FRICTION_IMPULSE:_abi.ST_FRICTION_IMPULSE + 4])
    on_bound = (lam_n > 1e-4) & (np.abs(lam_t - 0.1 * lam_n) <= 1e-6 * lam_n)
    assert on_bound.sum() > 100, on_bound.sum()
