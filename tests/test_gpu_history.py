# SPDX-License-Identifier: Apache-2.0
"""Spine-rate observation history on the device (upkie_b200_set_history): turning it on changes no output against a
FAM_SENSE twin, entry 0 is the tick's spine observation, entries move back by nb_substeps per tick, the entries match a
1 kHz handle's spine observations, resets of every kind fill the resetting envs only (sharded batches included), the
window follows the observation delay, the four vector envs expose it, checkpoints reproduce it, and the rejections."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, _abi
from test_gpu_observation_delay import _action, _bits, _config, _sim, _state, _step

pytestmark = pytest.mark.gpu

# 16 columns: base twist, pitch, IMU rate and both accelerations, a wheel's position / velocity / torque, odometry
COLS = ([_abi.SP_BASE_ANGVEL + 1, _abi.SP_BASE_LINVEL, _abi.SP_PITCH, _abi.SP_CONTACT]
        + list(range(_abi.SP_IMU_ANGVEL, _abi.SP_IMU_ANGVEL + 3)) + [_abi.SP_IMU_LINACC, _abi.SP_IMU_RAWACC + 2]
        + [_abi.SP_SERVO + 2 * 5 + k for k in range(3)] + [_abi.SP_SERVO + 1, _abi.SP_IMU_QUAT + 2]
        + [_abi.SP_ODOM_POS, _abi.SP_ODOM_VEL])
ACC = [c for c, col in enumerate(COLS) if _abi.SP_IMU_LINACC <= col < _abi.SP_IMU_RAWACC + 3]
NOACC = [c for c in range(len(COLS)) if c not in ACC]


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _hist(sim):
    return sim.get_history().cpu().numpy()


def _reset_envs(out, mode, prev_done):
    """the envs a step reset: the fused same-step resets of its terminal envs, the next-step resets of the previous
    step's"""
    done = (out[1] != 0) | (out[2] != 0)
    if mode == 2:
        return done, done
    if mode == 1:
        return prev_done, done
    return np.zeros_like(done), done


# ---- 1. no side effects --------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", ["servos", "pendulum"])
def test_history_changes_no_output(model, torch, kind, mode):
    n, T = 512, 60
    cfg = _config()
    hist = _sim(model, cfg, n, mode, sense=(0, 0), delay=(0, 3), push=True)
    hist.set_history(COLS, 40)
    twin = _sim(model, cfg, n, mode, sense=(0, 0), delay=(0, 3), push=True)
    resets = 0
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        out_h = _step(hist, kind, a, same_step=mode == 2)
        out_t = _step(twin, kind, a, same_step=mode == 2)
        for x, y in zip(out_h, out_t):
            assert (x is None) == (y is None)
            if x is not None:
                assert _bits(x) == _bits(y), k
        assert _bits(_state(hist)) == _bits(_state(twin)), k
        resets += int(((out_h[1] != 0) | (out_h[2] != 0)).sum())
    assert resets > 0
    for get in ("get_push_state", "get_action_delay_state", "get_observation_delay_state"):
        for x, y in zip(getattr(hist, get)(), getattr(twin, get)()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()), get


# ---- 2. / 3. entry 0 and the move across ticks --------------------------------------------------------------------


@pytest.mark.parametrize("mode", [1, 2])
def test_entry_zero_and_previous_ticks(model, torch, mode):
    n, T, K = 512, 30, 12
    cfg = _config()
    nb = cfg.nb_substeps
    sim = _sim(model, cfg, n, mode)
    sim.set_history(COLS, K)
    prev, prev_done, checked = None, np.zeros(n, bool), 0
    for k in range(T):
        out = _step(sim, "servos", _action(torch, model, "servos", n, k), same_step=mode == 2)
        h = _hist(sim)
        spine = out[5][:, COLS]
        # entry 0: the tick's spine observation, bit for bit (noise off), but the per-substep IMU accelerations
        np.testing.assert_array_equal(h[:, 0, NOACC], spine[:, NOACC])
        reset, prev_done = _reset_envs(out, mode, prev_done)
        if reset.any():  # a reset: every entry is the post-reset observation, accelerations included
            np.testing.assert_array_equal(h[reset], np.broadcast_to(spine[reset][:, None, :], h[reset].shape))
        if prev is not None:
            keep = ~reset
            np.testing.assert_array_equal(h[keep, nb:2 * nb], prev[keep, 0:nb])
            checked += int(keep.sum())
        prev = h
    assert checked > 0


# ---- 4. against a 1 kHz handle ------------------------------------------------------------------------------------


def test_entries_match_a_1khz_handle(model, torch):
    from upkie_b200.sim import UpkieSim

    n, K, ticks = 256, 5, 4
    cfg = _config(max_episode_steps=0, servos_fall_termination=0)
    fast = _config(max_episode_steps=0, servos_fall_termination=0, dt=0.001, nb_substeps=1)
    slow = UpkieSim(n, model=model, config=cfg)
    khz = UpkieSim(n, model=model, config=fast)
    slow.reset(seed=3)
    torch.cuda.synchronize()
    khz.set_state(slow.get_state())
    slow.set_history(COLS, K)
    a = _action(torch, model, "servos", n, 0)
    acc_err = 0.0
    for t in range(ticks):
        slow.step_servos(a)
        rows = []
        for _ in range(cfg.nb_substeps):
            khz.step_servos(a)
            rows.append(khz.spine_obs()[:, COLS].cpu().numpy())
        h = _hist(slow)
        for k in range(K):
            ref = rows[cfg.nb_substeps - 1 - k]
            np.testing.assert_allclose(h[:, k, NOACC], ref[:, NOACC], rtol=1e-5, atol=1e-5, err_msg=f"{t} {k}")
            # the accelerations differentiate velocities over 1 ms: their round-off is 1000 times the velocities'
            np.testing.assert_allclose(h[:, k, ACC], ref[:, ACC], rtol=1e-4, atol=2e-3, err_msg=f"{t} {k}")
            acc_err = max(acc_err, float(np.abs(h[:, k, ACC] - ref[:, ACC]).max()))
    assert np.abs(h[:, :, ACC]).max() > 0.1  # the accelerations are not trivially zero


# ---- 5. resets ----------------------------------------------------------------------------------------------------


def test_explicit_and_masked_resets_fill_only_their_envs(model, torch):
    n, K = 256, 9
    cfg = _config()
    sim = _sim(model, cfg, n, 0)
    sim.set_history(COLS, K)
    for k in range(6):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    before = _hist(sim)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    sim.reset(mask=mask, seed=SEED_MASK)
    torch.cuda.synchronize()
    after = _hist(sim)
    spine = sim.spine_obs()[:, COLS].cpu().numpy()
    m = mask.cpu().numpy().astype(bool)
    np.testing.assert_array_equal(after[m], np.broadcast_to(spine[m][:, None, :], after[m].shape))
    np.testing.assert_array_equal(after[~m], before[~m])
    sim.reset(seed=SEED_MASK + 1)  # all envs
    torch.cuda.synchronize()
    after = _hist(sim)
    spine = sim.spine_obs()[:, COLS].cpu().numpy()
    np.testing.assert_array_equal(after, np.broadcast_to(spine[:, None, :], after.shape))


SEED_MASK = 77


@pytest.mark.parametrize("mode", [1, 2])
def test_sharded_batches_match_the_whole(model, torch, mode):
    n, T, K = 512, 30, 7
    cfg = _config()
    whole = _sim(model, cfg, n, mode)
    parts = [_sim(model, cfg, n // 2, mode, env_offset=o) for o in (0, n // 2)]
    for s in [whole] + parts:
        s.set_history(COLS, K)
    for k in range(T):
        _step(whole, "servos", _action(torch, model, "servos", n, k), same_step=mode == 2)
        for o, s in zip((0, n // 2), parts):
            _step(s, "servos", _action(torch, model, "servos", n // 2, k, env_offset=o, total=n), same_step=mode == 2)
        hw = _hist(whole)
        assert _bits(hw[: n // 2]) == _bits(_hist(parts[0])), k
        assert _bits(hw[n // 2:]) == _bits(_hist(parts[1])), k


# ---- 6. observation delay -----------------------------------------------------------------------------------------


@pytest.mark.parametrize("d", [0, 1, 3, 5, 7, 10])
def test_entry_zero_is_the_delayed_observation(model, torch, d):
    n, T, K = 256, 25, 6
    cfg = _config()
    sim = _sim(model, cfg, n, 1)
    sim.set_history(COLS, K)  # before the delay: the delay's depth resizes the ring
    sim.set_observation_delay(d, d, max_ticks=2)
    sim.reset(seed=SEED_MASK)
    torch.cuda.synchronize()
    assert sim.history_entries() == K + 2 * cfg.nb_substeps
    torque = [c for c in NOACC if _abi.SP_SERVO <= COLS[c] < _abi.SP_ODOM_POS and (COLS[c] - _abi.SP_SERVO) % 5 == 2]
    for k in range(T):
        out = _step(sim, "servos", _action(torch, model, "servos", n, k))
        h = _hist(sim)
        spine = out[5][:, COLS]
        cols = [c for c in NOACC if c not in torque]
        np.testing.assert_array_equal(h[:, 0, cols], spine[:, cols], err_msg=str(k))
        # the delayed observation's torques are the snapshot's commanded torques: the substep's, noise off
        np.testing.assert_array_equal(h[:, 0, torque], spine[:, torque], err_msg=str(k))


# ---- 7. the four env types, checkpoints ---------------------------------------------------------------------------


@pytest.mark.parametrize("autoreset_mode", ["next_step", "same_step"])
@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_envs_expose_the_history(model, torch, env_type, autoreset_mode):
    from upkie_b200.envs import B200VectorEnv

    n, K = 64, 8
    keys = [("imu", "angular_velocity"), ("base_orientation", "pitch"), ("servo", "left_wheel", "velocity"),
            ("floor_contact", "contact")]
    env = B200VectorEnv(n, env_type=env_type, autoreset_mode=autoreset_mode, history=keys, history_size=K,
                        max_episode_steps=15)
    env.reset(seed=4)
    dim = {"servos": None, "gyropod": 2, "pendulum": 1, "base_velocity": 2}[env_type]
    for k in range(20):
        if dim is None:
            a = env.get_neutral_action()
            a = {j: {kk: np.broadcast_to(np.asarray(v, dtype=np.float32), (n,)).copy() for kk, v in d.items()}
                 for j, d in a.items()}
        else:
            a = np.random.default_rng(k).uniform(-0.5, 0.5, (n, dim)).astype(np.float32)
        _, _, _, _, info = env.step(a)
        so = info["spine_observation"]
        h = so.history
        assert tuple(h.shape) == (n, K, 3 + 1 + 1 + 1)
        arr = so.array
        np.testing.assert_array_equal(h[:, 0, :3].cpu().numpy(), arr[:, _abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3])
        np.testing.assert_array_equal(h[:, 0, 3].cpu().numpy(), arr[:, _abi.SP_PITCH])
        d0 = so[0]["history"]
        assert len(d0["imu"]["angular_velocity"]) == K and len(d0["imu"]["angular_velocity"][0]) == 3
        assert d0["base_orientation"]["pitch"][0] == so[0]["base_orientation"]["pitch"]
        assert isinstance(d0["floor_contact"]["contact"][0], bool)
        assert d0["servo"]["left_wheel"]["velocity"][0] == so[0]["servo"]["left_wheel"]["velocity"]
        if "final_info" in info:
            assert "history" not in info["final_info"]["spine_observation"][int(np.argmax(info["_final_info"]))]
    env.set_history(None)
    _, _, _, _, info = env.step(a)
    with pytest.raises(UpkieException):
        info["spine_observation"].history
    env.close()


def test_checkpoint_reproduces_the_next_histories(model, torch):
    n, K = 256, 11
    cfg = _config()
    a_sim = _sim(model, cfg, n, 2, delay=(0, 3), push=True)
    a_sim.set_observation_delay(0, 7, max_ticks=2)
    a_sim.set_history(COLS, K)
    a_sim.reset(seed=SEED_MASK)  # draws every env's observation delay
    for k in range(10):
        _step(a_sim, "servos", _action(torch, model, "servos", n, k), same_step=True)
    sd = a_sim.state_dict()
    b_sim = _sim(model, cfg, n, 2)
    b_sim.load_state_dict(sd)
    assert b_sim.history_spec == a_sim.history_spec
    for k in range(10, 30):
        a = _action(torch, model, "servos", n, k)
        x = _step(a_sim, "servos", a, same_step=True)
        y = _step(b_sim, "servos", a, same_step=True)
        assert _bits(x[0]) == _bits(y[0]), k
        assert _bits(_hist(a_sim)) == _bits(_hist(b_sim)), k


# ---- 8. rejections ------------------------------------------------------------------------------------------------


def test_rejections_keep_the_previous_spec(model, torch):
    from upkie_b200.sim import UpkieSim

    sim = _sim(model, _config(), 64, 1)
    sim.set_history(COLS[:4], 5)
    good = _hist(sim)
    for cols, size in ((COLS[:4], 0), (COLS[:4], 65), ([], 5), (COLS + [0], 5), ([62], 5), ([-1], 5)):
        with pytest.raises(UpkieException):
            sim.set_history(cols, size)
    assert sim.history_spec == (tuple(COLS[:4]), 5)
    assert _bits(_hist(sim)) == _bits(good)
    for kw in (dict(joint_limits=0), dict(body_contacts=1)):
        s = UpkieSim(64, model=model, config=_config(**kw))
        with pytest.raises(UpkieException, match="history"):
            s.set_history(COLS[:4], 5)
    with pytest.raises(UpkieException, match="history"):
        sim.set_config(_config(joint_limits=0))
    with pytest.raises(UpkieException, match="history"):
        sim.set_config(_config(body_contacts=1))
    s = UpkieSim(64, model=model, config=_config(spine_mode=1))
    with pytest.raises(UpkieException, match="spine_mode"):
        s.set_history(COLS[:4], 5)
    sim.set_history(None)
    with pytest.raises(UpkieException):
        sim.get_history()
