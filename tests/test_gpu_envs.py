# SPDX-License-Identifier: Apache-2.0
"""GPU tests through the C ABI: wrappers, reset, auto-reset, vector-env API, MPC,
full-size invariants."""
import numpy as np
import pytest

from conftest import mpc_kkt_residual, random_servo_actions, random_states
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _sim(n, model, cfg=None):
    from upkie_b200.sim import UpkieSim

    return UpkieSim(n, model=model, config=cfg if cfg is not None else _abi.default_sim_config())


def test_loaded_library_is_the_in_tree_cuda_build():
    from upkie_b200 import _lib

    assert _lib.LIB_PATH.endswith("upkie_b200/libupkie_b200.so")
    with open("/proc/self/maps") as f:
        _lib.lib()
        assert any("libupkie_b200.so" in line for line in f.read().splitlines())


def test_reset_matches_oracle(model, oracle_lib, torch):
    n = 1024
    cfg = _abi.default_sim_config()
    cfg.rand_pitch, cfg.rand_roll, cfg.rand_z, cfg.rand_omega_y = 0.3, 0.1, 0.05, 0.5
    rng = np.random.default_rng(0)
    init = np.stack([oracle_lib.sample_init_state(cfg, np.random.default_rng(s)) for s in range(n)]).astype(np.float32)
    init[:, 13:19] = rng.uniform(-0.3, 0.3, (n, 6))
    sim = _sim(n, model, cfg)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
    sim.reset(init_state=torch.from_numpy(init).cuda())
    osim.reset(init.astype(np.float64))
    gs, os_ = sim.get_state().cpu().numpy().astype(np.float64), osim.get_state()
    assert np.abs(gs[:, :7] - os_[:, :7]).max() < 1e-6
    assert np.abs(gs[:, 7:13] - os_[:, 7:13]).max() < 2e-3  # one substep of gravity/contact
    assert np.allclose(gs[:, 34:38], gs[:, [13, 14, 16, 17]])  # UpkieGyropod.reset leg targets
    for dim in (30, 6, 4):
        g = sim.reset_obs(dim).cpu().numpy().astype(np.float64).reshape(n, -1)
        o = osim.reset_obs(dim).reshape(n, -1)
        assert np.median(np.abs(g - o)) < 1e-5 and np.abs(g - o).max() < 5e-2
    # masked reset leaves the other envs untouched
    before = sim.get_state().clone()
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::2] = 1
    sim.reset(mask=mask, init_state=torch.from_numpy(init).cuda())
    after = sim.get_state()
    assert torch.equal(after[1::2], before[1::2])


def test_device_reset_starts_from_the_nominal_state(model, torch):
    """Auto-reset episodes (on-device sampler) start from the same state as ``reset()`` episodes: with the random
    bounds at zero, a reset sampled on the device equals a reset from the RobotState row, crouched joints and nominal
    base velocities included (round-1 advisor finding); ``update_init_rand`` reaches the device sampler."""
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.robot_state import RobotState, RobotStateRandomization

    crouch = np.array([0.4, -0.8, 0.0, -0.4, 0.8, 0.0])
    nominal = RobotState(joint_configuration=crouch, position_base_in_world=np.array([0.0, 0.0, 0.55]),
                         angular_velocity_base_in_base=np.array([0.0, 0.2, 0.0]),
                         linear_velocity_base_to_world_in_world=np.array([0.3, 0.0, 0.0]),
                         randomization=RobotStateRandomization())
    n = 256
    env = B200VectorEnv(n, "servos", model=model, init_state=nominal, autoreset_mode="next_step")
    env.sim.reset(seed=5)  # sampled on the device
    dev_state = env.sim.get_state().cpu().numpy()
    row = torch.from_numpy(np.tile(nominal.to_row().astype(np.float32), (n, 1))).cuda()
    env.sim.reset(init_state=row)
    row_state = env.sim.get_state().cpu().numpy()
    # identical up to the IMU finite-difference acceleration (columns 41:44), which spans the two resets because the
    # backend's previous IMU velocity survives a reset (pybullet_backend.py:220-267 does not clear it)
    keep = [c for c in range(_abi.STATE_DIM) if not 41 <= c < 44]
    assert np.array_equal(row_state[:, keep], dev_state[:, keep])
    assert np.abs(dev_state[:, 13:19] - crouch).max() < 5e-3  # one substep away from the nominal configuration
    # a fused auto-reset (next step after `terminated`) lands there too
    env.update_init_rand(pitch=0.25)
    env.sim.reset(seed=6)
    st = env.sim.get_state().cpu().numpy()
    pitch = 2 * np.arctan2(st[:, 5], st[:, 3])
    assert 0.05 < np.abs(pitch).max() <= 0.27 and pitch.std() > 0.08  # the new bound reached the device sampler
    assert np.abs(st[:, 13:19] - crouch).max() < 5e-3
    env.close()


def test_gyropod_and_pendulum_match_oracle(model, oracle_lib, torch):
    n = 1024
    cfg = _abi.default_sim_config()
    sim = _sim(n, model, cfg)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
    rng = np.random.default_rng(5)
    init = np.zeros((n, _abi.INIT_DIM), dtype=np.float32)
    init[:, 2] = 0.6
    pitch = rng.uniform(-0.3, 0.3, n)
    init[:, 3], init[:, 5] = np.cos(pitch / 2), np.sin(pitch / 2)
    sim.reset(init_state=torch.from_numpy(init).cuda())
    osim.reset(init.astype(np.float64))
    mism = 0
    for t in range(30):
        a = rng.uniform(-3.5, 3.5, (n, 2)).astype(np.float32)
        osim.set_state(sim.get_state().cpu().numpy().astype(np.float64))  # re-synchronise every tick
        g6, grew, gterm, gtrunc = sim.step_gyropod(torch.from_numpy(a).cuda())
        o6, orew, oterm, otrunc = osim.step_gyropod(a.astype(np.float64), 2)
        g6 = g6.cpu().numpy().astype(np.float64)
        assert np.abs(g6[:, [0, 1, 2, 5]] - o6[:, [0, 1, 2, 5]]).max() < 2e-4
        assert np.median(np.abs(g6[:, 3:5] - o6[:, 3:5])) < 1e-3
        safe = np.abs(np.abs(o6[:, 1]) - 1.0) > 1e-4
        assert np.array_equal(gterm.cpu().numpy()[safe], oterm[safe])
        mism += int((gterm.cpu().numpy()[~safe] != oterm[~safe]).sum())
        assert not gtrunc.any().item() and (grew == 0).all().item()
    assert mism <= 2
    a1 = rng.uniform(-3, 3, (n, 1)).astype(np.float32)
    osim.set_state(sim.get_state().cpu().numpy().astype(np.float64))
    g4, _, _, _ = sim.step_pendulum(torch.from_numpy(a1).cuda())
    o4, _, _, _ = osim.step_gyropod(a1.astype(np.float64), 1)
    assert np.abs(g4.cpu().numpy()[:, :2] - o4[:, :2]).max() < 2e-4


def test_randomization_matches_oracle(model, oracle_lib, torch):
    n = 1024
    cfg = _abi.default_sim_config()
    sim = _sim(n, model, cfg)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
    rng = np.random.default_rng(2)
    eps = rng.uniform(-0.2, 0.2, (n, 6)).astype(np.float32)
    mu = rng.uniform(0.5, 1.2, n).astype(np.float32)
    sim.set_randomization(friction=torch.from_numpy(mu).cuda(), inertia_eps=torch.from_numpy(eps).cuda())
    osim.set_randomization(friction=mu.astype(np.float64), inertia_eps=eps.astype(np.float64))
    st = random_states(n, seed=21).astype(np.float32)
    act = random_servo_actions(n, model, seed=22, torque_mode=True).astype(np.float32)
    sim.set_state(torch.from_numpy(st).cuda())
    osim.set_state(st.astype(np.float64))
    sim.step_servos(torch.from_numpy(act).cuda())
    osim.step_servos(act.astype(np.float64))
    gs, os_ = sim.get_state().cpu().numpy().astype(np.float64), osim.get_state()
    assert np.abs(gs[:, :7] - os_[:, :7]).max() < 2e-5
    assert np.median(np.abs(gs[:, 19:25] - os_[:, 19:25]).max(axis=1)) < 1e-3


@pytest.mark.parametrize("n", [4096, 1003])
def test_host_buffer_api_equals_device_api(model, torch, n):
    """Pinned buffers: the kernel reads / writes host memory itself (zero-copy, one launch); pageable buffers:
    staged chunks. Both must be bit-identical to the device-buffer call, full and partial warps alike."""
    a = random_servo_actions(n, model, seed=1).astype(np.float32)
    st = torch.from_numpy(random_states(n, seed=2).astype(np.float32)).cuda()
    s1, s2, s3 = _sim(n, model), _sim(n, model), _sim(n, model)
    for s in (s1, s2, s3):
        s.set_state(st)
    o1, r1, t1, u1 = s1.step_servos(torch.from_numpy(a).cuda())
    l0 = s2.launches
    pinned = s2.host_action_buffer(36)
    pinned[:] = a
    o2, r2, t2, u2 = s2.step_servos_host(pinned)  # zero-copy
    assert s2.launches - l0 == 1
    o3, r3, t3, u3 = s3.step_servos_host(a.copy())  # pageable action: staged
    # the pinned and the pageable route run the same TILE=1 kernel: bit-exact
    assert np.array_equal(o2, o3) and np.array_equal(t2, t3)
    # device buffers run the TILE=0 instantiation, compiled separately: same arithmetic, but the compiler is
    # free to contract / schedule it differently, so equality holds to round-off (amplified by the contact
    # rows' 1/h sensitivity on velocities), not bit for bit
    ref = o1.cpu().numpy()
    for o, r, t, u in ((o2, r2, t2, u2), (o3, r3, t3, u3)):
        d = np.abs(ref - o)
        # torques follow the joint rates through kd (x kd_scale up to 5): same round-off class as the velocities below
        assert d[:, :, 0].max() < 1e-5 and d[:, :, 2].max() < 1e-3 and np.median(d[:, :, 2]) < 1e-5, (
            d[:, :, 0].max(), d[:, :, 2].max())
        assert d[:, :, 1].max() < 2e-2 and np.median(d[:, :, 1]) < 1e-5, (d[:, :, 1].max(), np.median(d[:, :, 1]))
        assert np.array_equal(d[:, :, 3:], np.zeros_like(d[:, :, 3:]))
        assert np.array_equal(t1.cpu().numpy(), t) and np.array_equal(r1.cpu().numpy(), r)
        assert np.array_equal(u1.cpu().numpy(), u)
    # compact transport: only position / velocity / torque rows cross PCIe
    s4, s5 = _sim(n, model), _sim(n, model)
    s4.set_state(st)
    s5.set_state(st)
    p4 = s4.host_action_buffer(36)
    p4[:] = a
    c4, ct4 = s4.step_servos_host_compact(p4)
    c5, ct5 = s5.step_servos_host_compact(a.copy())  # pageable: staged through the handle's pinned buffers
    s6 = _sim(n, model)
    s6.set_state(st)
    c6, ct6 = s6.step_servos_compact(torch.from_numpy(a).cuda())  # device buffers, same TILE=1 kernel
    assert np.array_equal(c6.cpu().numpy(), c4) and np.array_equal(ct6.cpu().numpy(), ct4)
    for c, ct in ((c4, ct4), (c5, ct5)):
        assert c.shape == (n, 6, 3) and np.array_equal(c, o2[:, :, :3]) and np.array_equal(ct, t2)  # TILE=1 both
    g = np.random.default_rng(3).uniform(-3, 3, (n, 2)).astype(np.float32)
    o1, _, t1, _ = s1.step_gyropod(torch.from_numpy(g).cuda())
    pg = s2.host_action_buffer(2)
    pg[:] = g
    o2, _, t2, _ = s2.step_gyropod_host(pg)
    o3, _, t3, _ = s3.step_gyropod_host(g)
    assert np.array_equal(o2, o3) and np.array_equal(t2, t3)
    assert np.abs(o1.cpu().numpy() - o2).max() < 2e-2 and np.median(np.abs(o1.cpu().numpy() - o2)) < 1e-5
    assert np.array_equal(t1.cpu().numpy(), t2)
    p = np.random.default_rng(4).uniform(-3, 3, (n, 1)).astype(np.float32)
    o1, _, t1, _ = s1.step_pendulum(torch.from_numpy(p).cuda())
    pp = s2.host_action_buffer(1)
    pp[:] = p
    o2, _, t2, _ = s2.step_gyropod_host(pp)
    assert np.abs(o1.cpu().numpy() - o2).max() < 2e-2 and np.median(np.abs(o1.cpu().numpy() - o2)) < 1e-5
    assert np.array_equal(t1.cpu().numpy(), t2)


def test_vector_env_api_and_reference_semantics(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.robot_state import RobotState, RobotStateRandomization

    n = 64
    init = RobotState(randomization=RobotStateRandomization(pitch=0.2, z=0.05))
    env = B200VectorEnv(n, "servos", model=model, init_state=init)
    obs, info = env.reset(seed=42)
    assert set(obs) == set(_abi.JOINT_NAMES) and obs["left_hip"]["position"].shape == (n, 1)
    assert obs["left_hip"]["position"].dtype == np.float32
    assert np.all(obs["right_wheel"]["temperature"] == 42.0) and np.all(obs["right_wheel"]["voltage"] == 18.0)
    sp0 = info["spine_observation"][0]
    assert set(sp0) == {"base_orientation", "floor_contact", "imu", "servo", "wheel_odometry"}
    # seeding: env i draws from default_rng(seed + i), as UpkieEnv.reset(seed) would (upkie_env.py:180-190)
    obs_b, info_b = env.reset(seed=42)
    sa, sb = info["spine_observation"].array, info_b["spine_observation"].array
    # everything but the IMU accelerations repeats: the reference does NOT reset
    # __previous_imu_linear_velocity on reset (pybullet_backend.py:157,220-232), and neither do we
    keep = [i for i in range(_abi.SPINE_DIM) if not (_abi.SP_IMU_LINACC <= i < _abi.SP_IMU_RAWACC + 3)]
    assert np.array_equal(sa[:, keep], sb[:, keep])
    expect_pitch = [init.sample_state(np.random.default_rng(42 + i)).to_row()[3:7] for i in range(n)]
    st = env.sim.get_state().cpu().numpy()
    got_pitch = 2 * np.arctan2(st[:, 5], st[:, 3])
    want_pitch = np.array([2 * np.arctan2(q[2], q[0]) for q in expect_pitch])
    assert np.abs(got_pitch - want_pitch).max() < 2e-3  # one 1 ms substep after the reset
    action = {name: {"position": np.zeros((n, 1), np.float32), "velocity": np.zeros((n, 1), np.float32)}
              for name in ("left_hip", "left_knee", "right_hip", "right_knee")}
    obs, rew, term, trunc, info = env.step(action)
    assert rew.shape == (n,) and (rew == 0.0).all()  # upkie_env.py:230
    assert term.dtype == bool and not term.any() and not trunc.any()  # UpkieServos never terminates
    flat = np.zeros((n, 6, 6), np.float32)
    flat[:, :, 0] = np.nan
    obs2, *_ = env.step(flat)
    assert obs2["left_hip"]["torque"].shape == (n, 1)
    env.close()

    penv = B200VectorEnv(n, "pendulum", model=model)
    o, _ = penv.reset(seed=0)
    assert o.shape == (n, 4) and o.dtype == np.float32
    o, r, te, tr, _ = penv.step(np.zeros((n, 1), np.float32))
    assert o.shape == (n, 4) and penv.single_observation_space.shape == (4,)
    # README policy keeps every env up for a second (README.md:62-64)
    for _ in range(200):
        a = (10.0 * o[:, 0] + 1.0 * o[:, 1] + 0.0 * o[:, 2] + 0.1 * o[:, 3]).reshape(n, 1).astype(np.float32)
        o, r, te, tr, _ = penv.step(a)
        assert not te.any()
    assert np.abs(o[:, 0]).max() < 0.3
    # without control the robot falls and `terminated` is raised, and stays up to the user to reset
    fell = np.zeros(n, bool)
    for _ in range(400):
        o, r, te, tr, _ = penv.step(np.zeros((n, 1), np.float32))
        fell |= te
    assert fell.all()
    penv.close()


def test_autoreset_modes(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.robot_state import RobotState, RobotStateRandomization

    n = 256
    init = RobotState(randomization=RobotStateRandomization(pitch=0.4))
    zero = torch.zeros((n, 1), device="cuda")
    for mode in ("next_step", "same_step"):
        env = B200VectorEnv(n, "pendulum", model=model, init_state=init, autoreset_mode=mode)
        env.reset(seed=7)
        total_done, after_done_pitch = 0, []
        prev_term = torch.zeros(n, dtype=torch.uint8, device="cuda")
        for _ in range(600):
            o, r, te, tr, _ = env.step_tensors(zero)
            if mode == "next_step":
                # the step after a termination returns the reset observation with terminated = 0
                idx = prev_term.bool()
                if idx.any():
                    assert not te[idx].any().item()
                    after_done_pitch.append(o[idx, 0].abs().max().item())
            else:
                idx = te.bool()
                if idx.any():
                    after_done_pitch.append(o[idx, 0].abs().max().item())
            prev_term = te.clone()
            total_done += int(te.sum().item())
        assert total_done >= n  # every env fell at least once on average and kept running
        assert max(after_done_pitch) <= 0.4 + 0.05  # reset observations: |pitch| within the sampling bounds
        st = env.sim.get_state()
        assert torch.isfinite(st).all().item()
        env.close()


def test_env_index_sharding_is_invariant(model, torch):
    """Two shards of n/2 envs with env_offset reproduce one batch of n envs bit for bit
    (SURVEY.md 8e: results invariant to the GPU count)."""
    from upkie_b200 import _abi as A

    n = 512
    cfg = A.default_sim_config()
    cfg.rand_pitch, cfg.rand_omega_y = 0.3, 0.5
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    acts = torch.from_numpy(random_servo_actions(n, model, seed=3, torque_mode=True).astype(np.float32)).cuda()
    full = _sim(n, model, cfg)
    full.set_autoreset(1, 99, 0)
    full.reset(seed=99, env_offset=0)
    halves = []
    for k in range(2):
        h = _sim(n // 2, model, cfg)
        h.set_autoreset(1, 99, k * n // 2)
        h.reset(seed=99, env_offset=k * n // 2)
        halves.append(h)
    for t in range(60):
        of, _, tf, _ = full.step_servos(acts)
        parts = [h.step_servos(acts[k * n // 2:(k + 1) * n // 2].contiguous()) for k, h in enumerate(halves)]
        assert torch.equal(of, torch.cat([p[0] for p in parts]))
        assert torch.equal(tf, torch.cat([p[2] for p in parts]))
    assert torch.equal(full.get_state(), torch.cat([h.get_state() for h in halves]))


def test_mpc_matches_oracle(oracle_lib, torch):
    from upkie_b200.mpc import BatchedMPCBalancer

    for horizon in (16, 50):
        cfg = _abi.default_mpc_config()
        cfg.nb_timesteps = horizon
        n = 2048
        rng = np.random.default_rng(0)
        x0 = np.stack([rng.uniform(-0.5, 0.5, n), rng.uniform(-0.2, 0.2, n), rng.uniform(-0.5, 0.5, n),
                       rng.uniform(-1, 1, n)], 1).astype(np.float32)
        x0[:64, 1] = rng.uniform(0.3, 0.9, 64)
        x0[64:96, 1] = rng.uniform(1.05, 1.3, 32)
        vt = rng.uniform(-1, 1, n).astype(np.float32)
        contact = np.ones(n, np.uint8)
        contact[96:128] = 0
        mpc = BatchedMPCBalancer(n, config=cfg)
        v0 = rng.uniform(-1, 1, n).astype(np.float32)
        mpc.commanded_velocity.copy_(torch.from_numpy(v0).cuda())
        v = mpc.step_tensors(torch.from_numpy(x0).cuda(), torch.from_numpy(vt).cuda(), torch.from_numpy(contact).cuda(), 0.005)
        plan = mpc.plan().cpu().numpy().astype(np.float64)
        om = oracle_lib.OracleMpc(cfg)
        vc_o, first_o, found_o, plan_o = om.step(x0.astype(np.float64), vt.astype(np.float64), contact, 0.005,
                                                 v0.astype(np.float64), threads=8)
        assert mpc.found.all().item() and found_o.all()
        assert np.abs(plan[:, 0] - plan_o[:, 0]).max() < 1e-3  # |u0 - u0_oracle| <= ProxQP eps_abs (mpc_balancer.py:76)
        assert np.abs(plan - plan_o).max() < 5e-3
        assert np.abs(v.cpu().numpy() - vc_o).max() < 1e-5
        # accuracy gate of config 4 (SURVEY.md 8d): KKT residual of the device plan in the fp64 condensed QP
        Pm, _, _ = om.matrices()
        live = np.flatnonzero((np.abs(x0[:, 1]) <= 1.0) & (contact != 0))[:128]
        worst = max(mpc_kkt_residual(Pm, om.cost_vector(x0[i].astype(np.float64), float(vt[i])), plan[i], cfg.max_ground_accel)
                    for i in live)
        assert worst < 1e-3, worst
        assert np.abs(v.cpu().numpy()).max() <= 3.0
        # warm-started second tick stays consistent
        v2 = mpc.step_tensors(torch.from_numpy(x0).cuda(), torch.from_numpy(vt).cuda(), torch.from_numpy(contact).cuda(), 0.005)
        assert np.abs(mpc.plan().cpu().numpy() - plan_o).max() < 5e-3
        mpc.reset()
        assert (mpc.commanded_velocity == 0).all().item()


def test_mpc_in_the_loop_balances(model, torch):
    """UpkieBaseVelocity-style closed loop (upkie_base_velocity.py:164-202): MPC command -> gyropod env."""
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.mpc import BatchedMPCBalancer

    n = 128
    env = B200VectorEnv(n, "gyropod", model=model)
    env.reset(seed=1)
    mpc = BatchedMPCBalancer(n)
    target = torch.full((n,), 0.3, device="cuda")
    spine = env.sim.spine_obs()
    fell = torch.zeros(n, dtype=torch.bool, device="cuda")
    for _ in range(400):
        v = mpc.step_spine(target, spine, env.dt)
        a = torch.stack([v, torch.zeros_like(v)], dim=1).contiguous()
        o, r, te, tr, info = env.step_tensors(a)
        spine = env.sim.spine_obs()
        fell |= te.bool()
    assert not fell.any().item()
    assert (o[:, 3] - 0.3).abs().max().item() < 0.2  # tracks the commanded ground velocity
    assert o[:, 1].abs().max().item() < 0.3


def test_base_velocity_env(model, torch):
    """UpkieBaseVelocity semantics (tests/envs/test_upkie_base_velocity.py:35-105): zero observation at
    reset, SE(2) dead reckoning of the commanded velocity, balance kept by the embedded MPC."""
    import upkie_b200

    n = 64
    env = upkie_b200.make_vec("Upkie-B200-BaseVelocity", n, model=model)
    assert env.single_action_space.shape == (2,) and env.single_observation_space.shape == (3,)
    obs, info = env.reset(seed=3)
    assert obs.shape == (n, 3) and obs.dtype == np.float32 and not obs.any()
    a = np.tile(np.array([[0.2, 0.5]], dtype=np.float32), (n, 1))
    fell = np.zeros(n, bool)
    for k in range(300):
        obs, rew, term, trunc, info = env.step(a)
        fell |= term
    assert not fell.any()
    t = 300 * env.dt
    yaw = 0.5 * t  # yaw integrates the commanded yaw velocity
    assert np.allclose(obs[:, 2], yaw, atol=1e-3)
    # x = int v cos(psi) dt with psi the post-step yaw (upkie_base_velocity.py:197-199)
    k = np.arange(1, 301)
    x = (0.2 * np.cos(0.5 * k * env.dt) * env.dt).sum()
    y = (0.2 * np.sin(0.5 * k * env.dt) * env.dt).sum()
    assert np.allclose(obs[:, 0], x, atol=1e-4) and np.allclose(obs[:, 1], y, atol=1e-4)
    sp = info["spine_observation"].array
    assert np.abs(sp[:, _abi.SP_PITCH]).max() < 0.3
    obs, _ = env.reset(seed=3)
    assert not obs.any() and (env.mpc_balancer.commanded_velocity == 0).all().item()
    env.close()


def test_base_velocity_env_replays_the_reference_run(model, torch):
    """tests/golden/base_velocity_run.json - 300 ticks of the reference's own UpkieBaseVelocity env (MPCBalancer in
    front of the gyropod wrappers) on the oracle - replayed through B200VectorEnv on the GPU: same initial state and
    actions; the observation [x, y, yaw], the MPC's commanded ground velocity (which closes the loop through the
    simulated pitch / odometry) and `terminated` are compared tick by tick."""
    import json
    import os

    from upkie_b200.envs import B200VectorEnv

    run = json.load(open(os.path.join(os.path.dirname(__file__), "golden", "base_velocity_run.json")))
    n = 32  # identical copies: the batch must stay identical too
    env = B200VectorEnv(n, "base_velocity", model=model)
    row = torch.tensor(run["init_row"], dtype=torch.float32, device="cuda").reshape(1, -1).repeat(n, 1).contiguous()
    env.sim.reset(init_state=row)
    env.mpc_balancer.reset()
    env._xy.zero_()
    env._spine = env.sim.spine_obs()
    worst_obs, worst_v = 0.0, 0.0
    for t, (a, o, term, v) in enumerate(zip(run["actions"], run["obs"], run["terminated"], run["commanded_velocity"])):
        act = torch.tensor([a], dtype=torch.float32, device="cuda").repeat(n, 1).contiguous()
        obs, rew, te, tr, info = env.step(act)
        ob = obs.cpu().numpy()
        vc = env.mpc_balancer.commanded_velocity.cpu().numpy()
        assert np.array_equal(ob, np.tile(ob[:1], (n, 1))) and np.array_equal(vc, np.tile(vc[:1], n))
        worst_obs = max(worst_obs, float(np.abs(ob[0] - np.asarray(o)).max()))
        worst_v = max(worst_v, abs(float(vc[0]) - v))
        assert bool(te[0].item()) == term and float(rew[0].item()) == 0.0
    assert worst_obs < 5e-5, worst_obs  # dead reckoning of the commanded velocity along the post-step yaw
    assert worst_v < 2e-2, worst_v      # fp32 closed loop over 1.5 s against the fp64 run of the reference's classes
    env.close()


def test_full_size_invariants(model, torch):
    """BASELINE-size batch (65536 envs): finite state, unit quaternions, contact physics sane,
    reward/truncated constants, idempotent spine observation."""
    n = 65536
    cfg = _abi.default_sim_config()
    cfg.rand_pitch = 0.3
    sim = _sim(n, model, cfg)
    sim.reset(seed=5)
    a = torch.zeros((n, 6, 6), device="cuda")
    a[:, :, 0] = float("nan")
    a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    gen = torch.Generator(device="cuda")
    gen.manual_seed(0)
    for _ in range(40):
        a[:, :, 2] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * a[:, :, 5] * 0.2
        obs, rew, term, trunc = sim.step_servos(a)
    st = sim.get_state()
    assert torch.isfinite(st).all().item()
    assert (st[:, 3:7].norm(dim=1) - 1).abs().max().item() < 1e-5
    assert (rew == 0).all().item() and not trunc.any().item() and not term.any().item()
    assert (st[:, 19:25].abs() <= 100.0 + 1e-3).all().item()  # max coordinate velocity clamp
    on_ground = st[:, 40] > 0.5
    assert on_ground.float().mean().item() > 0.5
    s1, s2 = sim.spine_obs(), sim.spine_obs()
    assert torch.equal(s1, s2)  # observation has no side effects
    assert torch.equal(s1[:, 30:60].reshape(n, 6, 5), obs)
    assert (sim.error_flags() & 2).sum().item() == 0


def test_torque_noise_models(model, torch):
    """The FAM_EXTRAS instantiation of the step kernel: same draws as the CPU build of the same code (keyed on
    seed, global env index, per-env tick), reproducible, invariant to sharding, inert at sigma = 0."""
    from hostsim_wrap import HostSim
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.model import JointProperties

    n = 2048
    cfg = _abi.default_sim_config()
    for j in range(6):
        cfg.torque_control_noise[j] = (0.05, 0.0, 0.02)[j % 3]
        cfg.torque_measurement_noise[j] = (0.0, 0.03, 0.01)[j % 3]
    cfg.noise_seed = 99
    st = random_states(n, seed=3, z_range=(2.0, 3.0)).astype(np.float32)
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 2] = 0.5 * np.asarray(model.tau_max, dtype=np.float32)
    act[:, :, 5] = model.tau_max
    sim = _sim(n, model, cfg)
    sim.set_state(torch.from_numpy(st).cuda())
    hs = HostSim(model, cfg, n)
    hs.set_state(st)
    a = torch.from_numpy(act).cuda()
    for tick in (1, 2, 3):
        obs = sim.step_servos(a)[0].cpu().numpy()
        ref = hs.step_servos_noise(act, tick=tick)
        # torques depend on the noise only (pure feedforward): fast-math logf/sincosf vs libm
        assert np.abs(obs[:, :, 2] - ref[:, :, 2]).max() < 2e-5
        applied = sim.get_state()[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6].cpu().numpy()
        assert np.abs(applied - hs.state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6]).max() < 2e-5
        assert (obs[:, 1, 2] != applied[:, 1]).mean() > 0.99  # measurement noise on knees
        assert np.array_equal(obs[:, 0, 2], applied[:, 0])  # none on hips
    spine = sim.spine_obs().cpu().numpy()[:, _abi.SP_SERVO:_abi.SP_SERVO + 30].reshape(n, 6, 5)
    assert np.array_equal(spine[:, :, 2], obs[:, :, 2])  # the spine view repeats the step's draw

    # reproducible for a given seed, different for another one, invariant to the sharding of the env index
    def run(seed, offset=0, count=n):
        c = _abi.default_sim_config()
        for j in range(6):
            c.torque_control_noise[j] = 0.05
        c.noise_seed = seed
        s = _sim(count, model, c)
        s.set_autoreset(0, 0, offset)  # global env index of local env 0
        s.set_state(torch.from_numpy(st[offset:offset + count]).cuda())
        out = [s.step_servos(a[offset:offset + count])[0].clone() for _ in range(3)]
        return torch.stack(out).cpu().numpy()

    r1, r2, r3 = run(5), run(5), run(6)
    assert np.array_equal(r1, r2) and not np.array_equal(r1, r3)
    half = run(5, offset=n // 2, count=n // 2)
    assert np.array_equal(half, r1[:, n // 2:])

    # JointProperties through the env constructor; sigma = 0 is bit-identical to the default path
    props = {name: JointProperties(friction=0.0, torque_control_noise=0.0) for name in _abi.JOINT_NAMES}
    e0 = B200VectorEnv(64, "servos", model=model, joint_properties=props)
    e1 = B200VectorEnv(64, "servos", model=model)
    e0.reset(seed=1)
    e1.reset(seed=1)
    a64 = torch.from_numpy(act[:64]).cuda()
    assert torch.equal(e0.sim.step_servos(a64)[0], e1.sim.step_servos(a64)[0])
    noisy = {name: JointProperties(torque_control_noise=0.1, torque_measurement_noise=0.1) for name in _abi.JOINT_NAMES}
    e2 = B200VectorEnv(64, "servos", model=model, joint_properties=noisy, noise_seed=3)
    assert e2.config.torque_control_noise[2] == 0.1 and e2.config.noise_seed == 3
    e2.reset(seed=1)
    o2 = e2.sim.step_servos(torch.from_numpy(act[:64]).cuda())[0]
    assert not torch.equal(o2[:, :, 2], e1.sim.step_servos(torch.from_numpy(act[:64]).cuda())[0][:, :, 2])


def test_external_forces_and_imu_uncertainty(model, oracle_lib, torch):
    """External forces through the C ABI against the oracle's native formulation (free flight), their
    persistence / clearing, and ImuUncertainty on the spine observation."""
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.model import ExternalForce

    n = 1024
    cfg = _abi.default_sim_config()
    rng = np.random.default_rng(31)
    st = random_states(n, seed=32, z_range=(2.0, 3.0)).astype(np.float32)
    ext = rng.uniform(-20.0, 20.0, (n, 7, 3)).astype(np.float32)
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 2] = rng.uniform(-0.5, 0.5, (n, 6)) * model.tau_max
    act[:, :, 5] = 0.99 * np.asarray(model.tau_max, dtype=np.float32)
    a = torch.from_numpy(act).cuda()
    for mask in (0, 0b1001001):
        sim = _sim(n, model, cfg)
        osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
        sim.set_state(torch.from_numpy(st).cuda())
        osim.set_state(st.astype(np.float64))
        sim.set_external_forces(torch.from_numpy(ext).cuda(), mask)
        osim.set_external_forces(ext.astype(np.float64), mask)
        for _ in range(2):  # forces persist across steps
            sim.step_servos(a)
            osim.step_servos(act.astype(np.float64))
        d = np.abs(sim.get_state().cpu().numpy()[:, :25].astype(np.float64) - osim.get_state()[:, :25])
        assert d[:, :7].max() < 5e-6 and d[:, 13:19].max() < 5e-5
        assert d[:, 7:13].max() < 1e-3 and d[:, 19:25].max() < 1e-2
    # cleared forces: back to the plain kernel, bit-identical to a handle that never had any
    s1, s2 = _sim(n, model, cfg), _sim(n, model, cfg)
    for s in (s1, s2):
        s.set_state(torch.from_numpy(st).cuda())
    s1.set_external_forces(torch.from_numpy(ext).cuda(), 0)
    s1.set_external_forces(None)
    assert torch.equal(s1.step_servos(a)[0], s2.step_servos(a)[0])

    # env-level API: a sideways push on the torso of every other env, robots in free flight at rest
    env = B200VectorEnv(64, "servos", model=model)
    env.reset(seed=3)
    s0 = env.sim.get_state().clone()
    s0[:, _abi.ST_POS + 2] = 3.0
    s0[:, _abi.ST_LINVEL:_abi.ST_LINVEL + 6] = 0.0
    s0[:, _abi.ST_QD:_abi.ST_QD + 6] = 0.0
    env.sim.set_state(s0)
    push = np.zeros((64, 3))
    push[::2, 1] = 30.0
    env.set_external_forces({"torso": ExternalForce(push)})
    zero = torch.zeros((64, 6, 6), device="cuda")
    zero[:, :, 0] = float("nan")
    for _ in range(20):
        env.sim.step_servos(zero)
    vy = env.sim.get_state()[:, _abi.ST_LINVEL + 1].cpu().numpy()
    com_speed = 30.0 * 0.1 / float(np.sum(model.mass))  # F t / m at the robot's centre of mass; the base origin
    # also picks up the roll the off-centre push induces
    assert (vy[::2] > 0.5 * com_speed).all() and (vy[::2] < 3.0 * com_speed).all() and (np.abs(vy[1::2]) < 1e-4).all()
    env.set_external_forces(None)

    # ImuUncertainty (ImuUncertainty.h:63-69): bias + white noise on the IMU part of the spine observation only
    cfg2 = _abi.default_sim_config()
    cfg2.imu_accelerometer_bias[0], cfg2.imu_accelerometer_noise = 0.3, 0.05
    cfg2.imu_gyroscope_bias[2], cfg2.imu_gyroscope_noise = -0.1, 0.02
    cfg2.noise_seed = 4
    sa, sb = _sim(n, model, cfg2), _sim(n, model, cfg)
    for s in (sa, sb):
        s.set_state(torch.from_numpy(st).cuda())
        s.step_servos(a)
    pa, pb = sa.spine_obs().cpu().numpy(), sb.spine_obs().cpu().numpy()
    assert np.array_equal(sa.get_state().cpu().numpy(), sb.get_state().cpu().numpy())  # the physics is untouched
    other = np.ones(_abi.SPINE_DIM, dtype=bool)
    other[_abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3] = False
    other[_abi.SP_IMU_LINACC:_abi.SP_IMU_RAWACC + 3] = False
    assert np.array_equal(pa[:, other], pb[:, other])
    dacc = pa[:, _abi.SP_IMU_LINACC:_abi.SP_IMU_LINACC + 3] - pb[:, _abi.SP_IMU_LINACC:_abi.SP_IMU_LINACC + 3]
    draw = pa[:, _abi.SP_IMU_RAWACC:_abi.SP_IMU_RAWACC + 3] - pb[:, _abi.SP_IMU_RAWACC:_abi.SP_IMU_RAWACC + 3]
    dgyr = pa[:, _abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3] - pb[:, _abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3]
    for d_, bias, sig in ((dacc, [0.3, 0, 0], 0.05), (draw, [0.3, 0, 0], 0.05), (dgyr, [0, 0, -0.1], 0.02)):
        assert np.abs(d_.mean(axis=0) - bias).max() < 5 * sig / np.sqrt(n)
        assert np.abs(d_.std(axis=0) / sig - 1).max() < 0.1
    assert abs(np.corrcoef(dacc[:, 0], draw[:, 0])[0, 1]) < 0.12  # independent draws for the raw acceleration
    assert np.array_equal(sa.spine_obs().cpu().numpy(), pa)  # same tick, same draw


def test_checkpoint_resume_is_bit_exact(model, torch, tmp_path):
    """state_dict / load_state_dict: a fresh handle restored from a checkpoint continues bit for bit, with fused
    auto-resets (episode counters), torque noise (tick counters), randomisation and external forces in play."""
    n = 2048
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    for j in range(6):
        cfg.torque_control_noise[j] = 0.05
    cfg.noise_seed = 11
    rng = np.random.default_rng(5)
    act = np.zeros((n, 6, 6), dtype=np.float32)
    act[:, :, 0] = np.nan
    act[:, :, 2] = rng.uniform(-1, 1, (n, 6)) * model.tau_max
    act[:, :, 5] = model.tau_max
    a = torch.from_numpy(act).cuda()

    def fresh():
        return _sim(n, model, cfg)

    s1 = fresh()
    s1.set_randomization(torch.from_numpy(rng.uniform(0.5, 1.2, n).astype(np.float32)).cuda(),
                         torch.from_numpy(rng.uniform(-0.2, 0.2, (n, 6)).astype(np.float32)).cuda())
    ext = np.zeros((n, 7, 3), dtype=np.float32)
    ext[:, 0, 0] = 3.0
    s1.set_external_forces(torch.from_numpy(ext).cuda(), 0)
    s1.set_autoreset(1, 77, 0)
    s1.reset(seed=77)
    resets = 0
    for _ in range(150):
        resets += int(s1.step_servos(a)[2].sum().item())
    assert resets > 50  # the checkpoint is taken in the middle of resets
    path = tmp_path / "ckpt.pt"
    torch.save(s1.state_dict(), path)
    ref = [tuple(x.clone() for x in s1.step_servos(a)) for _ in range(40)]
    s2 = fresh()
    s2.load_state_dict(torch.load(path))
    for k in range(40):
        out = s2.step_servos(a)
        for x, y in zip(out, ref[k]):
            assert torch.equal(x, y), k
    assert torch.equal(s1.get_state(), s2.get_state())
