# SPDX-License-Identifier: Apache-2.0
"""Spine mode (config.spine_mode): the timing of the C++ Bullet spine in simulate() mode, rows a15 / f1 of SURVEY.md
section 8 - upkie/cpp/spine/Spine.cpp:116-140,185-265 (which observation a step returns),
upkie/cpp/interfaces/BulletInterface.cpp:129-163,228-352 (reset, cycle, torque law), bullet/read_imu_data.h:25-89.

CPU: the oracle's restatement is checked against the semantics read off the reference (black-box, through its public
state accessors), then the kernels' fp32 arithmetic (host build) against the oracle. GPU: the FAM_SPINE kernels through
the C ABI against the oracle."""
import numpy as np
import pytest

from conftest import random_servo_actions
from upkie_b200 import _abi


def _cfg(nb_substeps=5, frequency=200.0):
    cfg = _abi.default_sim_config(frequency)
    cfg.nb_substeps = nb_substeps
    cfg.spine_mode = 1
    return cfg


def _init(n, seed=0):
    rng = np.random.default_rng(seed)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2] = 0.58
    pitch = rng.uniform(-0.2, 0.2, n)
    init[:, 3], init[:, 5] = np.cos(pitch / 2), np.sin(pitch / 2)
    init[:, 10:13] = rng.uniform(-0.5, 0.5, (n, 3))  # angular_velocity_base_in_base
    init[:, 13:19] = rng.uniform(-0.3, 0.3, (n, 6))
    return init


def _servo_q(rows):
    return rows[:, _abi.SP_SERVO:_abi.SP_SERVO + 30:5]


def test_observation_lag_of_the_spine(model, oracle_lib):
    """With S physics steps done before an agent step, the observation holds the joint sensors of the state after S - 2
    steps and the IMU of the state after S - 1 steps (Spine.h:121-126 and the trace in DESIGN.md section 8); the reset
    runs three cycles and returns joints of step 0, IMU of step 1. One cycle per agent step (nb_substeps = 1) so that
    every intermediate state is visible through get_state()."""
    n = 64
    cfg = _cfg(nb_substeps=1, frequency=1000.0)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=2)
    init = _init(n)
    osim.reset(init.astype(np.float64))
    row0 = osim.spine_obs()
    assert np.abs(_servo_q(row0) - init[:, 13:19]).max() < 1e-7  # joints of step 0 = the reset configuration
    assert np.array_equal(row0[:, _abi.SP_SERVO + 3], np.full(n, 20.0)) and np.array_equal(row0[:, _abi.SP_SERVO + 4], np.full(n, 18.0))
    assert np.all(row0[:, _abi.SP_SERVO + 1:_abi.SP_SERVO + 30:5] == 0.0)  # resetJointState zeroes the rates
    states = [osim.get_state()]  # X_3: the state after the reset's three cycles
    # the servos were stopped during the reset: the joints did not move (locked), the base fell for 3 ms
    assert np.abs(states[0][:, 13:19] - init[:, 13:19]).max() < 1e-9 and np.abs(states[0][:, 19:25]).max() < 1e-9
    # angular velocity of the initial state: base frame -> world frame (BulletInterface.cpp:146-152)
    act = random_servo_actions(n, model, seed=1)
    rows = []
    for k in range(1, 8):
        osim.step_servos(act)
        rows.append(osim.spine_obs())
        states.append(osim.get_state())  # X_{3 + k}
    for k in range(3, 8):  # observation of step k: joints of X_k, and X_k = states[k - 3]
        assert np.abs(_servo_q(rows[k - 1]) - states[k - 3][:, 13:19]).max() < 1e-12, k
        assert np.abs(rows[k - 1][:, _abi.SP_SERVO + 1:_abi.SP_SERVO + 30:5] - states[k - 3][:, 19:25]).max() < 1e-12
    # IMU of X_{k + 1} = states[k - 2]: compare the orientation through a side simulator put in that state
    side = oracle_lib.OracleSim(model, _abi.default_sim_config(1000.0), n, threads=2)
    for k in range(2, 8):
        side.set_state(states[k - 2])
        side_row = _observe(side)
        assert np.abs(np.abs(rows[k - 1][:, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4]) - np.abs(side_row[:, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4])).max() < 1e-9, k
        assert np.abs(rows[k - 1][:, _abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3] - side_row[:, _abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3]).max() < 1e-9
    # the "sim" ground truth in the row is the CURRENT state at observation time (BulletInterface::observe): X_{k + 2}
    for k in range(1, 8):
        R = rows[k - 1][:, _abi.SP_ROT:_abi.SP_ROT + 9]
        side.set_state(states[k - 1])
        assert np.abs(R - _observe(side)[:, _abi.SP_ROT:_abi.SP_ROT + 9]).max() < 1e-9


def _row_diff(a, b):
    """(worst difference of the position-like entries + velocities, worst difference of the IMU accelerations). The
    velocity-like entries (base twist, IMU rates, joint rates) carry the usual fp32 contact round-off (5e-4 class); the
    accelerations are velocity differences divided by the 1 ms cycle, which turns 1e-7 m/s into 1e-4 m/s^2."""
    d = np.abs(np.asarray(a, dtype=np.float64) - np.asarray(b, dtype=np.float64))
    acc = np.zeros(d.shape[1], bool)
    acc[_abi.SP_IMU_LINACC:_abi.SP_IMU_LINACC + 3] = True
    acc[_abi.SP_IMU_RAWACC:_abi.SP_IMU_RAWACC + 3] = True
    vel = np.zeros(d.shape[1], bool)
    vel[_abi.SP_BASE_ANGVEL:_abi.SP_BASE_ANGVEL + 6] = True
    vel[_abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3] = True
    vel[_abi.SP_SERVO + 1:_abi.SP_SERVO + 30:5] = True
    vel[_abi.SP_SERVO + 2:_abi.SP_SERVO + 30:5] = True  # torques follow the rates through kd
    vel[_abi.SP_ODOM_VEL] = True
    assert np.median(d[:, vel].max(axis=1)) < 5e-5 and np.percentile(d[:, vel].max(axis=1), 99) < 5e-3
    return d[:, ~(acc | vel)].max(), d[:, acc].max()


def _observe(sim):
    """Spine row of a PyBullet-mode side simulator for its current state (oracle_observe + spine_obs)."""
    from oracle import oracle as O

    O.lib().oracle_observe(sim._h)
    return sim.spine_obs()


def test_spine_torque_law_clamps_at_the_urdf_effort(model, oracle_lib):
    """tau_max = min(maximum_torque, URDF effort) and no joint friction (BulletInterface.cpp:329-352; the reference's
    ComputeJointFeedforwardTorque test, BulletInterfaceTest.cpp:121-190, gives 0.42 for a 0.42 feedforward)."""
    cfg = _cfg(nb_substeps=1, frequency=1000.0)
    cfg.joint_friction[0] = 0.5  # ignored by the spine's law
    cfg.skip_action_clamps = 1
    osim = oracle_lib.OracleSim(model, cfg, 1)
    init = np.zeros((1, _abi.INIT_DIM))
    init[0, 2], init[0, 3] = 2.0, 1.0
    osim.reset(init)
    act = np.zeros((1, 6, 6))
    act[:, :, 0] = np.nan
    act[:, :, 2] = 0.42
    act[:, :, 5] = 1000.0  # above every effort limit
    act[0, 1, 2] = 50.0    # knee feedforward above its 16 N m effort
    osim.step_servos(act)
    lag = osim.get_lag()[0]
    tq = lag[_abi.LAG_REPLY1 + 2:_abi.LAG_REPLY1 + 18:3]
    assert tq[0] == pytest.approx(0.42, abs=1e-12) and tq[2] == pytest.approx(0.42, abs=1e-12)
    assert tq[1] == pytest.approx(16.0, abs=1e-12)


def test_kernel_arithmetic_in_spine_mode_matches_the_oracle(model, oracle_lib):
    """Host build of the kernels' spine-mode code (reset_robot_spine / spine_cycle, csrc/sim_core.cuh) against the
    oracle, re-synchronised every tick like the other arithmetic tests."""
    from hostsim_wrap import HostSim

    n = 1024
    cfg = _cfg()
    hs, osim = HostSim(model, cfg, n), oracle_lib.OracleSim(model, cfg, n, threads=4)
    init = _init(n, seed=3)
    row_h = hs.reset_spine(init)
    osim.reset(init.astype(np.float64))
    rest, acc = _row_diff(row_h, osim.spine_obs())
    assert rest < 2e-5 and acc < 2e-3, (rest, acc)
    d0 = np.abs(hs.state[:, :25] - osim.get_state()[:, :25])
    assert d0[:, :7].max() < 1e-5 and d0[:, 7:13].max() < 1e-3 and d0[:, 13:25].max() < 1e-6  # joints locked: exact
    act = random_servo_actions(n, model, seed=4).astype(np.float32)
    for tick in range(6):
        row_h = hs.step_servos_spine(act)
        osim.step_servos(act.astype(np.float64))
        row_o, st_o, lag_o = osim.spine_obs(), osim.get_state(), osim.get_lag()
        rest, acc = _row_diff(row_h, row_o)  # lagged rows: built from quantities both sides agreed on
        assert rest < 2e-4 and acc < 2e-2, (tick, rest, acc)
        d = np.abs(hs.state[:, :25].astype(np.float64) - st_o[:, :25])
        assert d[:, :7].max() < 2e-5 and d[:, 13:19].max() < 2e-4
        assert np.median(d[:, 19:25].max(axis=1)) < 5e-5 and np.percentile(d[:, 19:25].max(axis=1), 99) < 5e-3
        dl = np.abs(hs.lag[:, :49].astype(np.float64) - lag_o[:, :49])
        assert np.median(dl.max(axis=1)) < 1e-3
        osim.set_state(hs.state.astype(np.float64))
        lag = lag_o.copy()
        lag[:, :49] = hs.lag[:, :49]
        osim.set_lag(lag)


@pytest.mark.gpu
def test_spine_mode_on_device_matches_the_oracle(model, oracle_lib):
    import torch

    from upkie_b200.sim import UpkieSim

    n = 2048
    cfg = _cfg()
    sim, osim = UpkieSim(n, model=model, config=cfg), oracle_lib.OracleSim(model, cfg, n, threads=8)
    init = _init(n, seed=5)
    sim.reset(init_state=torch.from_numpy(init).cuda())
    osim.reset(init.astype(np.float64))
    rest, acc = _row_diff(sim.spine_obs().cpu().numpy(), osim.spine_obs())
    assert rest < 5e-5 and acc < 5e-3, (rest, acc)
    g30 = sim.reset_obs(30).cpu().numpy().reshape(n, 30)
    assert np.abs(g30 - osim.spine_obs()[:, _abi.SP_SERVO:_abi.SP_SERVO + 30]).max() < 1e-6
    act = random_servo_actions(n, model, seed=6).astype(np.float32)
    a = torch.from_numpy(act).cuda()
    for tick in range(5):
        gobs, _, gterm, _ = sim.step_servos(a)
        oobs, _, oterm, _ = osim.step_servos(act.astype(np.float64))
        g, o = gobs.cpu().numpy().reshape(n, 30), oobs.reshape(n, 30)
        assert np.abs(g - o).max() < 5e-4 and np.array_equal(g[:, 3::5], np.full((n, 6), 20.0, dtype=np.float32))
        rest, acc = _row_diff(sim.spine_obs().cpu().numpy(), osim.spine_obs())
        assert rest < 2e-4 and acc < 2e-2, (tick, rest, acc)
        gs, os_ = sim.get_state().cpu().numpy().astype(np.float64), osim.get_state()
        d = np.abs(gs[:, :25] - os_[:, :25])
        assert d[:, :7].max() < 2e-5 and d[:, 13:19].max() < 2e-4
        assert np.median(d[:, 19:25].max(axis=1)) < 5e-5 and np.percentile(d[:, 19:25].max(axis=1), 99) < 5e-3
        assert np.array_equal(gterm.cpu().numpy(), oterm)
        osim.set_state(gs)
        lag = osim.get_lag()
        lag[:, :49] = sim.get_lag().cpu().numpy()[:, :49]
        osim.set_lag(lag)


@pytest.mark.gpu
def test_spine_mode_vector_env_and_fused_autoreset(model):
    """B200VectorEnv(spine_mode=True): host path (TILE=1, FAM_SPINE kernel) and device path agree; a fused auto-reset
    runs the three stopped cycles and reports the reset configuration."""
    import torch

    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.robot_state import RobotState

    n = 256
    crouch = np.array([0.3, -0.6, 0.0, -0.3, 0.6, 0.0])
    nominal = RobotState(joint_configuration=crouch, position_base_in_world=np.array([0.0, 0.0, 0.56]))
    env = B200VectorEnv(n, "servos", model=model, spine_mode=True, init_state=nominal, autoreset_mode="next_step")
    env.config.servos_fall_termination = 1
    env.config.min_base_height = 0.3
    env.sim.set_config(env.config)
    obs, info = env.reset(seed=1)
    assert np.allclose(np.stack([obs[name]["position"][:, 0] for name in _abi.JOINT_NAMES], axis=1), crouch, atol=1e-6)
    assert float(obs["left_hip"]["temperature"][0, 0]) == 20.0
    act = env.sim.host_action_buffer()
    act[:] = 0.0
    act[:, :, 0] = np.nan  # no position target, no torque: the robots collapse and terminate on height
    seen_reset = np.zeros(n, bool)
    prev_term = np.zeros(n, bool)
    for k in range(120):
        obs, rew, term, trunc, info = env.step(act)
        q = np.stack([obs[name]["position"][:, 0] for name in _abi.JOINT_NAMES], axis=1)
        fresh = prev_term  # envs that terminated in the previous step were reset inside this one
        if fresh.any():
            assert np.allclose(q[fresh], crouch, atol=1e-6)  # observation of the reset: joints of step 0
            seen_reset |= fresh
        prev_term = term.copy()
    assert seen_reset.any()
    env.close()


@pytest.mark.gpu
def test_spine_pipeline_balances_on_lagged_observations(model):
    """The whole spine of `spines/bullet_spine.cpp --pipeline wheel_balancer` on the device, with the spine's timing:
    simulator in spine mode (one cycle per agent step at 1 kHz, `--nb-substeps 1`) -> lagged spine observation ->
    observer pipeline (BaseOrientation, FloorContact, WheelOdometry) -> WheelStopper + WheelBalancer -> servo action.
    Rows a14, a15, f1, f2 together: 256 robots started with up to 0.15 rad of pitch are upright after the transient."""
    import torch

    from upkie_b200.controllers import WheelBalancerPipeline
    from upkie_b200.observers import ObserverPipeline
    from upkie_b200.sim import UpkieSim

    n = 256
    cfg = _cfg(nb_substeps=1, frequency=1000.0)
    sim = UpkieSim(n, model=model, config=cfg)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2] = 0.58
    pitch0 = np.random.default_rng(3).uniform(-0.15, 0.15, n)
    init[:, 3], init[:, 5] = np.cos(pitch0 / 2), np.sin(pitch0 / 2)
    sim.reset(init_state=torch.from_numpy(init).cuda())
    obs_pipe = ObserverPipeline(n, model=model, spine_frequency=1000.0)
    wbc = _abi.default_wheel_balancer_config(1000.0)
    wbc.wheel_radius = float(model.wheel_radius)
    wb = WheelBalancerPipeline(n, config=wbc)
    neutral = torch.zeros((n, 6, 6), device="cuda")
    neutral[:, :, 3:5] = 1.0
    neutral[:, :, 5] = torch.tensor(model.tau_max, device="cuda", dtype=torch.float32)
    worst = []
    for k in range(3000):  # 3 s of spine cycles
        rows = obs_pipe.step(sim.spine_obs())  # the observation the spine assembled in its last cycle (lagged)
        act = wb.step(rows, neutral.clone())
        sim.step_servos(act)
        if k % 50 == 0:
            worst.append(rows[:, _abi.OBSV_PITCH].abs().max().item())
    st = sim.get_state().cpu().numpy()
    assert max(worst[20:]) < 0.3, max(worst[20:])
    assert (st[:, _abi.ST_POS + 2] > 0.4).all()


@pytest.mark.gpu
def test_peer_store_step_on_one_gpu_equals_the_compact_step(model):
    """`upkie_b200_step_servos_peers` (the in-kernel rollout transport without a multicast object) with this GPU's own
    buffer as the only "peer": same rows and `terminated` bytes as `upkie_b200_step_servos_compact`, bit for bit; two
    peers = two copies. (The multi-GPU form is validated by tools/multicast_check.py on 2 and 8 GPUs.)"""
    import torch

    from upkie_b200.sim import UpkieSim

    n = 4096
    cfg = _abi.default_sim_config()
    sims = [UpkieSim(n, model=model, config=cfg) for _ in range(2)]
    for s_ in sims:
        s_.reset(seed=4)
    act = torch.from_numpy(random_servo_actions(n, model, seed=9).astype(np.float32)).cuda()
    bufs = [torch.zeros(n * 18, dtype=torch.float32, device="cuda") for _ in range(2)]
    terms = [torch.zeros(n, dtype=torch.uint8, device="cuda") for _ in range(2)]
    for t in range(3):
        ref_obs, ref_term = sims[0].step_servos_compact(act)
        sims[1].step_servos_peers(act, [b.data_ptr() for b in bufs], [t_.data_ptr() for t_ in terms])
        torch.cuda.synchronize()
        # transport exact (both "peers" hold the same bytes); against the separately compiled TILE=1 kernel: round-off
        assert torch.equal(bufs[0], bufs[1]) and torch.equal(terms[0], terms[1])
        assert torch.allclose(bufs[0].view(n, 6, 3), ref_obs, rtol=0, atol=2e-2) and torch.equal(terms[0], ref_term)
        assert float((bufs[0].view(n, 6, 3) - ref_obs).abs().median()) < 1e-6


@pytest.mark.gpu
def test_deferred_push_on_one_gpu_equals_the_compact_step(model):
    """`upkie_b200_step_servos_push` / `upkie_b200_push_rows` (deferred rollout transport): every step writes its rows to
    a local slot and the NEXT launch's prologue copies them to the destination buffers (here: two local "peer" buffers);
    after the final `push_rows` the destinations hold the same rows as the compact step produced, slot by slot."""
    import torch

    from upkie_b200 import _abi as A
    from upkie_b200.sim import UpkieSim

    n, T = 4096, 4
    cfg = A.default_sim_config()
    sims = [UpkieSim(n, model=model, config=cfg) for _ in range(2)]
    for s_ in sims:
        s_.reset(seed=4)
    act = torch.from_numpy(random_servo_actions(n, model, seed=9).astype(np.float32)).cuda()
    local_obs = torch.zeros((T, n * 18), dtype=torch.float32, device="cuda")
    local_term = torch.zeros((T, n), dtype=torch.uint8, device="cuda")
    dst_obs = [torch.zeros((T, n * 18), dtype=torch.float32, device="cuda") for _ in range(2)]
    dst_term = [torch.zeros((T, n), dtype=torch.uint8, device="cuda") for _ in range(2)]
    ref = []

    def descriptor(t):
        d = A.UpkiePush()
        d.src_obs, d.src_terminated = local_obs[t].data_ptr(), local_term[t].data_ptr()
        for p in range(2):
            d.peer_obs[p], d.peer_terminated[p] = dst_obs[p][t].data_ptr(), dst_term[p][t].data_ptr()
        d.n_peers = 2
        return d

    pending = None
    for t in range(T):
        o, te = sims[0].step_servos_compact(act)
        ref.append((o.clone(), te.clone()))
        sims[1].step_servos_push(act, local_obs[t].data_ptr(), local_term[t].data_ptr(), pending)
        pending = descriptor(t)
        torch.cuda.synchronize()
        if t > 0:  # the previous step's rows arrived with this launch, this step's have not left yet
            assert torch.equal(dst_obs[0][t - 1], local_obs[t - 1]) and not dst_obs[0][t].any()
    sims[1].push_rows(pending)
    torch.cuda.synchronize()
    for t in range(T):
        for p in range(2):  # transport: byte for byte what the kernel wrote to its local slot
            assert torch.equal(dst_obs[p][t], local_obs[t]) and torch.equal(dst_term[p][t], local_term[t])
        # physics against the separately compiled TILE=1 kernel: fp32 round-off, same flags
        assert torch.allclose(local_obs[t].view(n, 6, 3), ref[t][0], rtol=0, atol=2e-2)
        assert float((local_obs[t].view(n, 6, 3) - ref[t][0]).abs().median()) < 1e-6 and torch.equal(local_term[t], ref[t][1])
