# SPDX-License-Identifier: Apache-2.0
"""IMU attitude estimation on the device (upkie_b200_set_attitude_filter): a filter turned off leaves a handle bit for
bit as one that never had it; an fp64 replay of the filter driven by each substep's history columns and the env's IMU
biases reproduces the reported estimates and the step's pitch, with and without a misalignment, under a one-tick
observation delay; the draws and the initial estimates of fused, explicit and seeded resets; the same-step final
observation; checkpoints and set_state; every output but the orientation is that of a twin without the filter; the
rejections."""
import numpy as np
import pytest
import torch as torch_mod
from scipy.spatial.transform import Rotation

from upkie_b200 import UpkieRuntimeError, _abi
from test_attitude_filter_cpu import RBI, draw_np, step_np

pytestmark = pytest.mark.gpu

SEED = 0x5151
NEXT_STEP, SAME_STEP = 1, 2
SPEC = ((1.0, 10.0), (0.0, 0.5), (-0.05, 0.05), (-0.05, 0.05))
HIST = [*range(_abi.SP_IMU_ANGVEL, _abi.SP_IMU_ANGVEL + 3), *range(_abi.SP_IMU_RAWACC, _abi.SP_IMU_RAWACC + 3),
        *range(_abi.SP_IMU_QUAT, _abi.SP_IMU_QUAT + 4), _abi.SP_PITCH]
ORIENT = [_abi.SP_PITCH, *range(_abi.SP_ROT, _abi.SP_IMU_ANGVEL)]
ARS = np.diag([1.0, -1.0, -1.0])


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _config(**kw):
    cfg = _abi.default_sim_config()
    cfg.rand_pitch = 0.1
    cfg.max_episode_steps = 60
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _sim(model, cfg, n, mode, att=SPEC, history=None, sense=None, tilt=None, bias=False, env_offset=0):
    """a handle reset once; a zero-probability servo-dropout spec runs it in FAM_SENSE, so that a twin without the
    filter runs the same kernels"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if bias:
        rows = s.get_env_params()
        g = torch_mod.Generator(device="cpu").manual_seed(3)
        rows[:, _abi.EP_IMU_GYRO_BIAS:_abi.EP_IMU_GYRO_BIAS + 3] = ((torch_mod.rand((n, 3), generator=g) * 2 - 1)
                                                                    * 0.02).cuda()
        rows[:, _abi.EP_IMU_ACC_BIAS:_abi.EP_IMU_ACC_BIAS + 3] = ((torch_mod.rand((n, 3), generator=g) * 2 - 1)
                                                                  * 0.1).cuda()
        s.set_env_params(rows.contiguous())
    if history:
        s.set_history(history, cfg.nb_substeps)
    if sense is not None:
        s.set_observation_delay(*sense)
    if tilt is not None:
        s.set_imu_misalignment(*tilt)
    s.set_servo_dropout(0.0, 0.0)
    if att is not None:
        s.set_attitude_filter(*att)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _policy(obs):
    """a balancing pendulum: ground velocity from pitch and pitch rate (obs [pitch, p, pitch rate, pdot])"""
    return (8.0 * obs[:, 0:1] + 0.8 * obs[:, 2:3]).clamp(-2.0, 2.0).contiguous()


def _np(x):
    return x.clone().cpu().numpy()


def _att(sim):
    return [_np(t).astype(np.float64) for t in sim.get_attitude_filter_state()]


def _pitch_of(q_iw):
    """the base pitch of estimates q_iw [n, 4] (IMU-to-world), taken back to the base through rotation_base_to_imu"""
    R = Rotation.from_quat(q_iw, scalar_first=True).as_matrix() @ RBI
    return np.arcsin(np.clip(-R[:, 2, 0], -1, 1))


def _from_ars(q_ars):
    """the IMU-to-world estimates of reported imu.orientation quaternions (ARS frame)"""
    R = ARS @ Rotation.from_quat(q_ars, scalar_first=True).as_matrix()
    return Rotation.from_matrix(R).as_quat(scalar_first=True)


def _qdist(a, b):
    return np.minimum(np.abs(a - b).max(axis=-1), np.abs(a + b).max(axis=-1))


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_off_is_bit_for_bit_a_handle_without_it(model, torch, mode):
    n = 256
    cfg = _config()
    a = _sim(model, cfg, n, mode, att=None, history=ORIENT)
    b = _sim(model, cfg, n, mode, att=SPEC, history=ORIENT)
    b.set_attitude_filter(None)
    b.reset(seed=SEED)
    a.reset(seed=SEED)
    obs_a = obs_b = torch.zeros((n, 4), device="cuda")
    for _ in range(40):
        oa, _, ta, ra = a.step_pendulum(_policy(obs_a))
        ob, _, tb, rb = b.step_pendulum(_policy(obs_b))
        for x, y in ((oa, ob), (ta, tb), (ra, rb), (a.spine_obs(), b.spine_obs()), (a.get_history(), b.get_history()),
                     (a.get_state(), b.get_state())):
            assert torch.equal(x, y)
        obs_a, obs_b = oa, ob


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_outputs_but_the_orientation_are_unaffected(model, torch, mode):
    n = 256
    cfg = _config()
    twin = _sim(model, cfg, n, mode, att=None, history=HIST, bias=True)
    sim = _sim(model, cfg, n, mode, history=HIST, bias=True)
    keep = [c for c in range(_abi.SPINE_DIM) if c not in ORIENT]
    hkeep = [k for k, c in enumerate(HIST) if c not in ORIENT]
    obs = torch.zeros((n, 4), device="cuda")
    for t in range(60):
        act = _policy(obs)  # the twin is driven by the filtered pitch too, so that both run the same physics
        ot, _, tt, rt = twin.step_pendulum(act)
        o, _, te, tr = sim.step_pendulum(act)
        assert torch.equal(o[:, 1:], ot[:, 1:]) and torch.equal(te, tt) and torch.equal(tr, rt)
        assert torch.equal(sim.get_state(), twin.get_state())
        assert torch.equal(sim.spine_obs()[:, keep], twin.spine_obs()[:, keep])
        assert torch.equal(sim.get_history()[:, :, hkeep], twin.get_history()[:, :, hkeep])
        obs = o
    assert not torch.equal(o[:, 0], ot[:, 0])  # the pitch is the estimate's


@pytest.mark.parametrize("tilt", [None, ((-0.05, 0.05), (-0.05, 0.05), (-0.1, 0.1))])
def test_fp64_replay_of_the_history_reproduces_the_estimates(model, torch, tilt):
    n, ticks = 512, 400
    cfg = _config(max_episode_steps=0)
    nb = cfg.nb_substeps
    h = cfg.dt / nb
    sim = _sim(model, cfg, n, NEXT_STEP, history=HIST, tilt=tilt, bias=True)
    ep = _np(sim.get_env_params()).astype(np.float64)
    gb = ep[:, _abi.EP_IMU_GYRO_BIAS:_abi.EP_IMU_GYRO_BIAS + 3]
    ab = ep[:, _abi.EP_IMU_ACC_BIAS:_abi.EP_IMU_ACC_BIAS + 3]
    obs = torch.zeros((n, 4), device="cuda")
    pending = np.zeros(n, dtype=bool)
    worst_q = worst_p = 0.0
    checked = 0
    for t in range(ticks):
        count0, gains, q0, b0 = _att(sim)
        obs, _, term, trunc = sim.step_pendulum(_policy(obs))
        hist = _np(sim.get_history()).astype(np.float64)  # [n, nb, C], newest first
        count1, _, q1, b1 = _att(sim)
        pitch = _np(obs[:, 0]).astype(np.float64)
        live = ~pending & (count1 == count0)
        pending = _np(term | trunc).astype(bool)
        for i in np.flatnonzero(live)[:64]:
            q, b = q0[i], b0[i]
            for s in range(nb):
                e = hist[i, nb - 1 - s]
                q, b = step_np(q, b, gains[i, 0], gains[i, 1], h, e[0:3] + gb[i], e[3:6] + ab[i])
                worst_q = max(worst_q, _qdist(_from_ars(e[6:10]), q))
            worst_q = max(worst_q, _qdist(q1[i], q), np.abs(b1[i] - b).max())
            worst_p = max(worst_p, abs(pitch[i] - _pitch_of(q[None])[0]), abs(hist[i, 0, 10] - pitch[i]))
            checked += 1
    assert checked > 0.9 * 64 * ticks
    assert worst_q < 2e-5, worst_q
    assert worst_p < 2e-5, worst_p


def test_one_tick_observation_delay_reports_the_observed_cycle(model, torch):
    n = 512
    cfg = _config(max_episode_steps=0)
    sim = _sim(model, cfg, n, NEXT_STEP, history=HIST, sense=(0, cfg.nb_substeps))
    obs = torch.zeros((n, 4), device="cuda")
    pending = np.zeros(n, dtype=bool)
    for t in range(100):
        obs, _, term, trunc = sim.step_pendulum(_policy(obs))
        hist = _np(sim.get_history()).astype(np.float64)  # entry 0: the observed instant
        spine = _np(sim.spine_obs()).astype(np.float64)
        live = ~pending
        pending = _np(term | trunc).astype(bool)
        est = _from_ars(hist[live, 0, 6:10])
        np.testing.assert_allclose(_np(obs[:, 0])[live], _pitch_of(est), atol=1e-5)
        np.testing.assert_allclose(spine[live, _abi.SP_PITCH], hist[live, 0, 10], atol=1e-5)
        assert np.all(_qdist(spine[live, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4], hist[live, 0, 6:10]) < 1e-5)


def _initial(qb, angles):
    """the estimate of a base observed with orientation qb and a drawn error (roll, pitch): qb E qbi^-1"""
    E = Rotation.from_euler("ZYX", np.stack([np.zeros(len(angles)), angles[:, 1], angles[:, 0]], 1))
    R = (Rotation.from_quat(qb, scalar_first=True) * E).as_matrix() @ RBI.T
    return Rotation.from_matrix(R).as_quat(scalar_first=True)


def _spec_struct():
    return _abi.UpkieAttitudeFilter(*(v for r in SPEC for v in r))


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_resets_draw_and_initialise(model, torch, mode):
    n, off = 256, 700
    cfg = _config(max_episode_steps=7)
    sim = _sim(model, cfg, n, mode, env_offset=off)
    g = off + np.arange(n, dtype=np.uint64)
    spec = _spec_struct()
    expect = np.ones(n, dtype=np.int64)
    pending = np.zeros(n, dtype=bool)
    obs = torch.zeros((n, 4), device="cuda")
    for k in range(30):
        count0, _, q0, _ = _att(sim)
        obs, _, term, trunc = sim.step_pendulum(_policy(obs))
        done = _np(term | trunc).astype(bool)
        reset_now = done if mode == SAME_STEP else pending
        expect += reset_now
        count, gains, quat, bias = _att(sim)
        np.testing.assert_array_equal(count, expect)
        d = draw_np(spec, SEED, g, expect)
        np.testing.assert_array_equal(gains[reset_now], d[reset_now, :2])
        if reset_now.any():
            qb = _np(sim.get_state())[reset_now, 3:7].astype(np.float64)
            assert np.all(_qdist(quat[reset_now], _initial(qb, d[reset_now, 2:4])) < 1e-5)
            assert np.all(bias[reset_now] == 0)
            np.testing.assert_allclose(_np(obs[:, 0])[reset_now], _pitch_of(quat[reset_now]), atol=1e-5)
        pending = done
    assert expect.max() > 3
    # explicit masked resets: only the masked envs draw
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    before = _att(sim)
    sim.reset(mask=mask, seed=SEED, env_offset=off)
    m = _np(mask).astype(bool)
    after = _att(sim)
    np.testing.assert_array_equal(after[0][~m], before[0][~m])
    for a, b in zip(after[1:], before[1:]):
        np.testing.assert_array_equal(a[~m], b[~m])
    np.testing.assert_array_equal(after[0][m], before[0][m] + 1)
    d = draw_np(spec, SEED, g, after[0].astype(np.int64))
    np.testing.assert_array_equal(after[1][m], d[m, :2])


def test_seeded_resets_repeat_and_draws_follow_the_global_index(model, torch):
    from upkie_b200.envs import B200VectorEnv

    att = {"kp": SPEC[0], "ki": SPEC[1], "roll": SPEC[2], "pitch": SPEC[3]}
    env = B200VectorEnv(64, env_type="pendulum", attitude_filter=att)
    env.reset(seed=11)
    first = _att(env.sim)
    for _ in range(5):
        env.step(np.zeros((64, 1), np.float32))
    env.reset(seed=11)
    again = _att(env.sim)
    for a, b in zip(first, again):
        np.testing.assert_array_equal(a, b)
    cfg = _config()
    whole = _sim(model, cfg, 64, NEXT_STEP)
    lo = _sim(model, cfg, 32, NEXT_STEP, env_offset=0)
    hi = _sim(model, cfg, 32, NEXT_STEP, env_offset=32)
    g_whole = _att(whole)[1]
    np.testing.assert_array_equal(g_whole, np.concatenate([_att(lo)[1], _att(hi)[1]]))


def test_checkpoint_continues_bit_for_bit_and_set_state_reinitialises(model, torch):
    n = 256
    cfg = _config()
    sim = _sim(model, cfg, n, SAME_STEP, history=HIST, sense=(0, 3), bias=True)
    obs = torch.zeros((n, 4), device="cuda")
    for _ in range(25):
        obs, *_ = sim.step_pendulum(_policy(obs))
    sd = sim.state_dict()
    assert "attitude_filter_quat" in sd
    other = _sim(model, cfg, n, SAME_STEP, att=None, history=HIST, sense=(0, 3), bias=True)
    other.load_state_dict(sd)
    o2 = obs.clone()
    for _ in range(20):
        obs, _, t1, _ = sim.step_pendulum(_policy(obs))
        o2, _, t2, _ = other.step_pendulum(_policy(o2))
        assert torch.equal(obs, o2) and torch.equal(t1, t2)
        assert torch.equal(sim.spine_obs(), other.spine_obs())
        for a, b in zip(sim.get_attitude_filter_state(), other.get_attitude_filter_state()):
            assert torch.equal(a, b)
    # set_state: every estimate restarts from the state set, without an error and without a bias estimate
    count, gains, _, _ = _att(sim)
    sim.set_state(sim.get_state())
    c2, g2, quat, bias = _att(sim)
    np.testing.assert_array_equal(c2, count)
    np.testing.assert_array_equal(g2, gains)
    assert np.all(bias == 0)
    qb = _np(sim.get_state())[:, 3:7].astype(np.float64)
    assert np.all(_qdist(quat, _initial(qb, np.zeros((n, 2)))) < 1e-5)
    # older checkpoints load with the filter off
    for k in [k for k in sd if k.startswith("attitude_filter")]:
        del sd[k]
    sim.load_state_dict(sd)
    assert sim.attitude_filter_spec is None


def test_rejections(model, torch):
    cfg = _config()
    sim = _sim(model, cfg, 64, NEXT_STEP, att=((1.0, 400.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0)))
    coarse = _config(nb_substeps=1)
    with pytest.raises(UpkieRuntimeError):
        sim.set_config(coarse)  # 400 * 5 ms > 0.5
    with pytest.raises(UpkieRuntimeError):
        sim.set_observation_delay(0, 7, max_ticks=2)
    sim.set_observation_delay(0, 3)  # one tick is fine
    for bad in (((1.0, 600.0),), ((1.0, 1.0), (0.0, 11.0)), ((1.0, 1.0), (0.0, 0.0), (0.0, 0.9))):
        with pytest.raises(UpkieRuntimeError):
            sim.set_attitude_filter(*bad)
    assert sim.attitude_filter_spec[0][1] == pytest.approx(400.0)
    count, gains, quat, bias = sim.get_attitude_filter_state()
    with pytest.raises(UpkieRuntimeError):
        sim.set_attitude_filter_state(count, gains, quat * 1.01, bias)
    with pytest.raises(UpkieRuntimeError):
        sim.set_attitude_filter_state(count, gains * 100.0, quat, bias)
    sim.set_attitude_filter(None)
    sim.set_observation_delay(0, 7, max_ticks=2)
    with pytest.raises(UpkieRuntimeError):
        sim.set_attitude_filter(*SPEC)  # the other order


@pytest.mark.parametrize("sense", [None, (0, 5)])
def test_same_step_final_observation_is_the_terminal_estimate(model, torch, sense):
    """A same-step handle's final observation and final spine observation of an env's first termination against a
    next-step twin, which runs the same ticks up to it and reports the terminal step as its ordinary observation (its
    reset waits for the next step). Under an observation delay the report is the snapshot's estimate, not the newest."""
    n = 256
    cfg = _config(max_episode_steps=15)
    same = _sim(model, cfg, n, SAME_STEP, sense=sense)
    nxt = _sim(model, cfg, n, NEXT_STEP, sense=sense)
    obs = torch.zeros((n, 4), device="cuda")
    seen = np.zeros(n, dtype=bool)
    for _ in range(15):
        act = _policy(obs)
        fin = torch.full((n, 4), float("nan"), device="cuda")
        obs, _, term, trunc = same.step_pendulum(act, final_obs=fin, final_state=True)
        fso = _np(same.final_spine_obs()).astype(np.float64)
        o_n, *_ = nxt.step_pendulum(act)
        first = _np(term | trunc).astype(bool) & ~seen
        if first.any():
            ref = _np(o_n).astype(np.float64)[first]
            np.testing.assert_allclose(_np(fin).astype(np.float64)[first], ref, atol=1e-5)
            spine = _np(nxt.spine_obs()).astype(np.float64)[first]
            np.testing.assert_allclose(fso[first][:, ORIENT], spine[:, ORIENT], atol=1e-5)
        seen |= first
    assert seen.all()


@pytest.mark.parametrize("order", ["on_after_step", "off_after_step"])
def test_spec_change_invalidates_the_final_stash(model, torch, order):
    n = 128
    cfg = _config(max_episode_steps=3)
    sim = _sim(model, cfg, n, SAME_STEP, att=None if order == "on_after_step" else SPEC)
    act = torch.zeros((n, 1), device="cuda")
    for _ in range(3):
        sim.step_pendulum(act, final_obs=torch.zeros((n, 4), device="cuda"), final_state=True)
    sim.final_spine_obs()  # valid: every env terminated in the last step
    if order == "on_after_step":
        sim.set_attitude_filter(*SPEC)
    else:
        sim.set_attitude_filter(None)
    with pytest.raises(UpkieRuntimeError):
        sim.final_spine_obs()
    # the next stashing step lays the stash out for the spec in force
    for _ in range(3):
        fin = torch.zeros((n, 4), device="cuda")
        sim.step_pendulum(act, final_obs=fin, final_state=True)
    fso = _np(sim.final_spine_obs()).astype(np.float64)
    np.testing.assert_allclose(fso[:, _abi.SP_PITCH], _np(fin[:, 0]), atol=1e-5)


def test_report_is_kept_by_masked_resets_and_checkpoints(model, torch):
    """Under a one-tick observation delay the report is the snapshot's estimate: restarting the draw counters of some
    envs (B200VectorEnv.reset's masked seeded reset) leaves the others' observations as they were, and a checkpoint
    carries it."""
    n = 128
    cfg = _config(max_episode_steps=0)
    sim = _sim(model, cfg, n, NEXT_STEP, sense=(5, 5), history=HIST)
    obs = torch.zeros((n, 4), device="cuda")
    for _ in range(20):
        obs, *_ = sim.step_pendulum(_policy(obs))
    before = sim.spine_obs().clone()
    rep = sim.get_attitude_filter_report()
    assert not torch.equal(rep, sim.get_attitude_filter_state()[2])  # a whole tick behind the estimate
    other = _sim(model, cfg, n, NEXT_STEP, att=None, sense=(5, 5), history=HIST)
    other.load_state_dict(sim.state_dict())
    assert torch.equal(other.spine_obs(), before)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::4] = 1
    count, gains, quat, bias = sim.get_attitude_filter_state()
    count.masked_fill_(mask.bool(), 0)
    sim.set_attitude_filter_state(count, gains, quat, bias)
    sim.reset(mask=mask, seed=7)
    keep = ~mask.bool()
    assert torch.equal(sim.spine_obs()[keep], before[keep])
    with pytest.raises(UpkieRuntimeError):
        sim.set_attitude_filter_report(rep * 1.01)


def test_set_config_checks_the_gains_envs_hold(model, torch):
    n = 64
    cfg = _config()
    sim = _sim(model, cfg, n, NEXT_STEP, att=((1.0, 400.0), (0.0, 0.0), (0.0, 0.0), (0.0, 0.0)))
    sim.set_attitude_filter((1.0, 10.0))  # the envs keep their gains up to 400 until their next reset
    coarse = _config(nb_substeps=1)
    with pytest.raises(UpkieRuntimeError):
        sim.set_config(coarse)
    sim.reset(seed=SEED)  # every env draws from (1, 10): 10 * 5 ms is within the bound
    sim.set_config(coarse)
