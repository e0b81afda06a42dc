# SPDX-License-Identifier: Apache-2.0
"""Observation-delay randomisation on the device (upkie_b200_set_observation_delay): a zero delay changes nothing
against the table and action-delay twins, the physics does not depend on the draws, the observation is the snapshot of
the state nb_substeps - d substeps into the tick with the IMU differentiated between snapshots, the draws and the
undelayed observation after fused, explicit, masked and sharded resets, the delayed terminal observations of same-step
resets, the four env types with pushes and the action delay, checkpoints, the rejections and a cleared spec."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_observation_delay_cpu import observation_delay_draw_np
from test_push_randomization_cpu import make_spec

pytestmark = pytest.mark.gpu

SEED = 31
PUSH = dict(gap=(0, 6), duration=(1, 5), force=((-30.0, -30.0, -5.0), (30.0, 30.0, 5.0)))
# the sensed columns of a state row, and among them the base pose / twist and joint columns
SENSED = [k for k in range(_abi.STATE_DIM)
          if k < _abi.ST_LEG_TARGET or k == _abi.ST_CONTACT or _abi.ST_IMU_ACC <= k < _abi.ST_IMU_ACC + 3]
BODY = list(range(_abi.ST_PREV_IMU_VEL)) + list(range(_abi.ST_TORQUE, _abi.ST_TORQUE + 6))
# the IMU velocity and acceleration columns of a state row, the IMU acceleration columns of a spine observation
IMU_ST = list(range(_abi.ST_PREV_IMU_VEL, _abi.ST_PREV_IMU_VEL + 3)) + list(range(_abi.ST_IMU_ACC, _abi.ST_IMU_ACC + 3))
IMU_ACC_SP = list(range(_abi.SP_IMU_LINACC, _abi.SP_IMU_RAWACC + 3))
# the columns of the gyropod and pendulum rows computed from the orientation: pitch and pitch rate
ORIENTATION_COLS = {"gyropod": [1, 4], "pendulum": [0, 2]}


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _config(**kw):
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.max_episode_steps = 20
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _sim(model, cfg, n, mode, sense=None, delay=None, push=False, env_offset=0, table=False):
    """a handle with the given ranges set, then reset once: the explicit reset draws every env's first delays"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if table:  # the config's values in a table: the FAM_TABLE kernels
        s.set_env_params(s.get_env_params())
    if push:
        s.set_push_randomization(make_spec(**PUSH))
    if delay is not None:
        s.set_action_delay(*delay)
    if sense is not None:
        s.set_observation_delay(*sense)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k, env_offset=0, total=None):
    total = total or n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(5000 + k)
    if kind == "servos":
        a = torch.zeros((total, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((total, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((total, 6), device="cuda", generator=gen) * 2 - 1) * 4.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    else:
        dim = 2 if kind == "gyropod" else 1
        a = (torch.rand((total, dim), device="cuda", generator=gen) * 2 - 1) * 2.0
    return a[env_offset : env_offset + n].contiguous()


FINAL_SHAPE = {"servos": (6, 5), "gyropod": (6,), "pendulum": (4,)}


def _step(sim, kind, a, same_step=False):
    """(obs, terminated, truncated, final_obs or None, final spine obs or None, spine obs) as NumPy arrays"""
    step = {"servos": sim.step_servos, "gyropod": sim.step_gyropod, "pendulum": sim.step_pendulum}[kind]
    fin = fso = None
    if same_step:
        fin = torch_mod.zeros((sim.n,) + FINAL_SHAPE[kind], device="cuda")
        obs, _, term, trunc = step(a, final_obs=fin, final_state=True)
        fso = sim.final_spine_obs()
    else:
        obs, _, term, trunc = step(a)
    out = [obs, term, trunc, fin, fso, sim.spine_obs()]
    return [None if x is None else x.clone().cpu().numpy() for x in out]


def _bits(x):
    return np.ascontiguousarray(x).tobytes()


def _state(sim):
    return sim.get_state().cpu().numpy()


def _rows(sim):
    return sim.get_observation_delay_state()[2].cpu().numpy()


# ---- 1. a zero delay changes nothing -----------------------------------------------------------------------------------


@pytest.mark.parametrize("action_delay", [False, True])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_zero_delay_matches_the_twin(model, torch, kind, mode, action_delay):
    n, T = 512, 60
    cfg = _config()
    delay = (0, 3) if action_delay else None
    sensed = _sim(model, cfg, n, mode, sense=(0, 0), delay=delay)
    twin = _sim(model, cfg, n, mode, delay=delay, table=not action_delay)  # FAM_DELAY or FAM_TABLE
    resets = 0
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        out_s = _step(sensed, kind, a, same_step=mode == 2)
        out_t = _step(twin, kind, a, same_step=mode == 2)
        # In the same-step gyropod and pendulum kernels fast-math contracts the products of the orientation into FMAs
        # in another order in FAM_SENSE than in FAM_TABLE (measured on an H100): the pitch and pitch rate of the rows,
        # and the IMU velocity of the state (hence the IMU acceleration), differ in the last bits on some envs. Neither
        # feeds back into the dynamics; every other field, output and state column matches bit for bit.
        contracted = kind != "servos" and mode == 2
        for j, (x, y) in enumerate(zip(out_s, out_t)):
            assert (x is None) == (y is None)
            if x is None:
                continue
            if contracted and j in (0, 3):
                cols = ORIENTATION_COLS[kind]
                x, y = x.reshape(n, -1), y.reshape(n, -1)
                # (the pitch rate sums three products of the orientation with the base rate: up to 1.2e-5 rad/s apart)
                np.testing.assert_allclose(x[:, cols], y[:, cols], rtol=1e-5, atol=5e-5, err_msg=str(k))
                assert _bits(np.delete(x, cols, axis=1)) == _bits(np.delete(y, cols, axis=1)), k
            elif contracted and j in (4, 5):
                np.testing.assert_allclose(x[:, IMU_ACC_SP], y[:, IMU_ACC_SP], rtol=1e-5, atol=1e-4, err_msg=str(k))
                assert _bits(np.delete(x, IMU_ACC_SP, axis=1)) == _bits(np.delete(y, IMU_ACC_SP, axis=1)), k
            else:
                assert _bits(x) == _bits(y), k
        resets += int(((out_s[1] != 0) | (out_s[2] != 0)).sum())
        xs, ys = _state(sensed), _state(twin)
        if contracted:
            # the acceleration differentiates the velocity over dt: its last bits are 200 times the velocity's
            np.testing.assert_allclose(xs[:, IMU_ST], ys[:, IMU_ST], rtol=1e-5, atol=1e-4, err_msg=str(k))
            xs, ys = np.delete(xs, IMU_ST, axis=1), np.delete(ys, IMU_ST, axis=1)
        assert _bits(xs) == _bits(ys), k
    assert resets > 0
    assert _bits(_rows(sensed)) == _bits(_state(sensed))  # d = 0: the sensed rows are the state


def test_zero_delay_host_path(model, torch):
    # The host-buffer (TILE=1) kernels of FAM_SENSE and FAM_TABLE are separately compiled copies of the same physics,
    # which can differ in the last bits within a tick (test_gpu_action_delay.py): the twin is put back on the delayed
    # handle's state before every tick, integer outputs bit for bit, observations within fp32 round-off of one tick.
    n, T = 512, 40
    cfg = _config()
    sensed = _sim(model, cfg, n, 2, sense=(0, 0))
    twin = _sim(model, cfg, n, 2, table=True)
    for k in range(T):
        a = _action(torch, model, "servos", n, k).cpu().numpy().reshape(n, 36)
        twin.set_state(sensed.get_state())
        torch.cuda.synchronize()
        x = [np.array(v, copy=True) for v in sensed.step_host(a, 36, compact=True, final_obs=True)]
        y = [np.array(v, copy=True) for v in twin.step_host(a, 36, compact=True, final_obs=True)]
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        np.testing.assert_allclose(x[0], y[0], rtol=1e-5, atol=1e-3, err_msg=str(k))
        done = (x[1] | x[2]).astype(bool)
        np.testing.assert_allclose(x[3][done], y[3][done], rtol=1e-5, atol=1e-3, err_msg=str(k))


# ---- 2. the physics does not depend on the draws -------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [1, 2])
def test_physics_is_independent_of_the_draws(model, torch, mode):
    n, T = 512, 60
    cfg = _config()
    a_sim = _sim(model, cfg, n, mode, sense=(0, 5), delay=(0, 2), push=True)
    b_sim = _sim(model, cfg, n, mode, sense=(0, 0), delay=(0, 2), push=True)
    differ = False
    for k in range(T):
        act = _action(torch, model, "gyropod", n, k)
        x = _step(a_sim, "gyropod", act)
        y = _step(b_sim, "gyropod", act)
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        assert _bits(_state(a_sim)) == _bits(_state(b_sim)), k
        assert torch.equal(a_sim.error_flags(), b_sim.error_flags())
        assert torch.equal(a_sim.get_push_forces(), b_sim.get_push_forces())
        differ |= _bits(x[0]) != _bits(y[0])
    assert differ  # the observations do see the delays
    assert a_sim.get_observation_delay_state()[1].any()


# ---- 3. the snapshot ---------------------------------------------------------------------------------------------------


def test_full_delay_reports_the_start_of_the_tick(model, torch):
    n, T, nb = 512, 20, 5
    cfg = _config(max_episode_steps=0, servos_fall_termination=0, nb_substeps=nb)
    sim = _sim(model, cfg, n, 0, sense=(nb, nb))
    sim.set_observation_delay_state(torch.zeros(n, dtype=torch.int32, device="cuda"),
                                    torch.full((n,), nb, dtype=torch.int32, device="cuda"), sim.get_state())
    for k in range(T):
        before = _state(sim)
        obs = _step(sim, "servos", _action(torch, model, "servos", n, k))[0]
        assert _bits(obs[:, :, 0]) == _bits(before[:, _abi.ST_Q:_abi.ST_Q + 6]), k
        assert _bits(obs[:, :, 1]) == _bits(before[:, _abi.ST_QD:_abi.ST_QD + 6]), k
        assert _bits(obs[:, :, 2]) == _bits(before[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6]), k
        assert _bits(_rows(sim)[:, BODY]) == _bits(before[:, BODY]), k
        assert _bits(_state(sim)) != _bits(before)


@pytest.mark.parametrize("d", [1, 2, 3, 4])
def test_partial_delay_matches_a_shorter_tick(model, torch, d):
    # a twin with the same substep length and nb - d substeps per tick, put on the same state before every tick
    n, T, nb = 512, 10, 5
    cfg = _config(max_episode_steps=0, servos_fall_termination=0, nb_substeps=nb)
    cfg_twin = _config(max_episode_steps=0, servos_fall_termination=0, nb_substeps=nb - d,
                       dt=cfg.dt * (nb - d) / nb)
    sim = _sim(model, cfg, n, 0, sense=(d, d), table=False)
    sim.set_observation_delay_state(torch.zeros(n, dtype=torch.int32, device="cuda"),
                                    torch.full((n,), d, dtype=torch.int32, device="cuda"), sim.get_state())
    twin = _sim(model, cfg_twin, n, 0, table=True)
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        twin.set_state(sim.get_state())
        torch.cuda.synchronize()
        x = _step(sim, "servos", a)
        y = _step(twin, "servos", a)
        assert _bits(x[0][:, :, :3]) == _bits(y[0][:, :, :3]), k
        assert _bits(_rows(sim)[:, BODY]) == _bits(_state(twin)[:, BODY]), k
        # spine observation: base orientation, twist and servo rows of the snapshot
        for cols in (slice(0, _abi.SP_IMU_QUAT), slice(_abi.SP_SERVO, _abi.SP_SERVO + 30)):
            assert _bits(x[5][:, cols]) == _bits(y[5][:, cols]), k


def test_imu_acceleration_differentiates_consecutive_snapshots(model, torch):
    n, T = 512, 30
    cfg = _config(max_episode_steps=0, servos_fall_termination=0)
    sim = _sim(model, cfg, n, 0, sense=(0, 5))
    sim.set_observation_delay_state(torch.zeros(n, dtype=torch.int32, device="cuda"),
                                    torch.arange(n, dtype=torch.int32, device="cuda") % 6, sim.get_state())
    prev = _rows(sim)
    inv_dt = np.float32(1.0 / cfg.dt)
    for k in range(T):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
        rows = _rows(sim)
        v, v0 = rows[:, _abi.ST_PREV_IMU_VEL:_abi.ST_PREV_IMU_VEL + 3], prev[:, _abi.ST_PREV_IMU_VEL:_abi.ST_PREV_IMU_VEL + 3]
        np.testing.assert_allclose(rows[:, _abi.ST_IMU_ACC:_abi.ST_IMU_ACC + 3], (v - v0) * inv_dt, rtol=1e-5, atol=1e-3)
        prev = rows


# ---- 4. resets ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "pendulum"])
@pytest.mark.parametrize("mode", [0, 1, 2])
def test_draws_and_reset_observations(model, torch, kind, mode):
    n, T, low, high = 1024, 120, 0, 5
    sim = _sim(model, _config(), n, mode, sense=(low, high))
    g = np.arange(n, dtype=np.uint64)
    expect = np.ones(n, dtype=np.uint64)  # the explicit reset after the spec: draw 1
    done_prev = np.zeros(n, dtype=bool)
    assert _bits(_rows(sim)) == _bits(_state(sim))  # the reset's observation is undelayed
    for k in range(T):
        out = _step(sim, kind, _action(torch, model, kind, n, k))
        done = (out[1] | out[2]).astype(bool)
        if mode:
            reset_now = done_prev if mode == 1 else done
            expect += reset_now.astype(np.uint64)
            # the envs that reset in this step observe their post-reset state
            rows, st = _rows(sim), _state(sim)
            assert _bits(rows[reset_now]) == _bits(st[reset_now]), k
        done_prev = done
    count, delay, _ = (x.cpu().numpy() for x in sim.get_observation_delay_state())
    np.testing.assert_array_equal(count.astype(np.uint64), expect)
    np.testing.assert_array_equal(delay.astype(np.uint32), observation_delay_draw_np(low, high, SEED, g, expect))
    if mode:
        assert expect.max() > 3
    # an explicit masked reset, with device-sampled and with host rows
    for init in (None, "host"):
        mask = ((np.arange(n) % 3) == (0 if init is None else 1)).astype(np.uint8)
        rows = None
        if init == "host":
            rows = torch.zeros((n, _abi.INIT_DIM), device="cuda")
            rows[:, 2] = 0.58
            rows[:, 3] = 1.0
        sim.reset(mask=torch.from_numpy(mask).cuda(), init_state=rows, seed=SEED)
        expect = expect + mask.astype(np.uint64)
        count, delay, srows = (x.cpu().numpy() for x in sim.get_observation_delay_state())
        np.testing.assert_array_equal(count.astype(np.uint64), expect)
        np.testing.assert_array_equal(delay.astype(np.uint32), observation_delay_draw_np(low, high, SEED, g, expect))
        sel = mask == 1
        assert _bits(srows[sel]) == _bits(_state(sim)[sel])


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 60
    whole = _sim(model, _config(), n, 2, sense=(0, 5))
    half = n // 2
    shards = [_sim(model, _config(), half, 2, sense=(0, 5), env_offset=o) for o in (0, half)]
    for k in range(T):
        out = _step(whole, "servos", _action(torch, model, "servos", n, k))
        for s, o in zip(shards, (0, half)):
            part = _step(s, "servos", _action(torch, model, "servos", half, k, env_offset=o, total=n))
            assert _bits(part[0]) == _bits(out[0][o : o + half])
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_observation_delay_state(), whole.get_observation_delay_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o : o + half])


@pytest.mark.parametrize("kind", ["servos", "gyropod"])
def test_same_step_terminal_observations_are_delayed(model, torch, kind):
    # d = nb: the terminal observation and its spine observation are those of the state before the step
    n, T, nb = 1024, 60, 5
    cfg = _config(nb_substeps=nb, max_episode_steps=7)
    sim = _sim(model, cfg, n, 2, sense=(nb, nb))
    twin = _sim(model, cfg, n, 0, table=True)  # spine observations of the states before the steps
    resets = 0
    for k in range(T):
        before = sim.get_state()
        twin.set_state(before)
        twin_spine = twin.spine_obs().cpu().numpy()
        before = before.cpu().numpy()
        out = _step(sim, kind, _action(torch, model, kind, n, k), same_step=True)
        done = (out[1] | out[2]).astype(bool)
        resets += int(done.sum())
        if kind == "servos":
            assert _bits(out[3][done][:, :, 0]) == _bits(before[done][:, _abi.ST_Q:_abi.ST_Q + 6]), k
            assert _bits(out[3][done][:, :, 1]) == _bits(before[done][:, _abi.ST_QD:_abi.ST_QD + 6]), k
        for cols in (slice(0, _abi.SP_IMU_QUAT), slice(_abi.SP_SERVO, _abi.SP_SERVO + 30)):
            assert _bits(out[4][done][:, cols]) == _bits(twin_spine[done][:, cols]), k
        # the reset observation is undelayed
        assert _bits(_rows(sim)[done]) == _bits(_state(sim)[done]), k
    assert resets > 0


# ---- 5. env types and interactions -------------------------------------------------------------------------------------


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import neutral_action

    n = 128
    push = {"link": "torso", "interval": (0.0, 0.05), "duration": (0.01, 0.03),
            "force": ((-40.0, -40.0, 0.0), (40.0, 40.0, 0.0))}
    dim = {"servos": None, "gyropod": 2, "pendulum": 1, "base_velocity": 2}[env_type]

    def run(env, reps=1):
        gen = torch.Generator(device="cuda")
        outs = []
        for _ in range(reps):
            env.reset(seed=5)
            gen.manual_seed(7)
            out = []
            for _ in range(40):
                if dim is None:
                    a = neutral_action(env.model, n, "cuda")
                    a[:, :, 1] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 3.0
                else:
                    a = (torch.rand((n, dim), device="cuda", generator=gen) * 2 - 1) * 0.5
                obs, _, term, trunc, _ = env.step_tensors(a)
                out.append((obs.clone(), term.clone(), env.sim.get_state().clone()))
            outs.append(out)
        return outs

    kw = dict(autoreset_mode="next_step", max_episode_steps=25, push_randomization=push, action_delay=(0.0, 0.002))
    env = B200VectorEnv(n, env_type, observation_delay=(0.001, 0.005), **kw)
    assert env.sim._observation_delay == (1, 5)  # 1 ms substeps at 200 Hz
    first, second = run(env, 2)
    count, _, _ = (x.cpu().numpy() for x in env.sim.get_observation_delay_state())
    assert np.all(count >= 1)
    env.reset(seed=5)
    delay = env.sim.get_observation_delay_state()[1].cpu().numpy()  # the first draws, those of step 0
    # reset(seed) restarts the draws: the runs repeat, but for the first observation of the envs that report the
    # start of the tick (d = nb_substeps): its torques are the ones the state held at the reset, which the reset leaves
    # as the earlier run left them (the reference's __joint_torques, pybullet_backend.py:163,294)
    for k, (x, y) in enumerate(zip(first, second)):
        for j, (u, v) in enumerate(zip(x, y)):
            if k == 0 and j == 0:
                full = torch.from_numpy(delay == 5).to(u.device)
                u, v = u[~full], v[~full]
            assert torch.equal(torch.nan_to_num(u, nan=1e30), torch.nan_to_num(v, nan=1e30)), (k, j)
    # against the same env without the delay: the same physics and terminations, other observations
    plain = B200VectorEnv(n, env_type, **kw)
    (other,) = run(plain)
    seen = False
    for k, (x, y) in enumerate(zip(first, other)):
        # base_velocity's observation (x, y, yaw) is dead-reckoned from its commands and the wrapper's yaw: the delay
        # shows in its physics, through the MPC reading the delayed spine observation
        seen |= not torch.equal(x[2] if env_type == "base_velocity" else x[0], y[2] if env_type == "base_velocity" else y[0])
        if env_type != "base_velocity" and k < 10:  # base_velocity's actions depend on the observations
            # separately compiled copies of the physics (FAM_SENSE, FAM_DELAY): equal up to fp32 round-off
            assert torch.equal(x[1], y[1]), k
            torch.testing.assert_close(x[2], y[2], rtol=1e-4, atol=1e-4)
    assert seen
    env.set_observation_delay(None)
    assert env.sim._observation_delay is None
    with pytest.raises(UpkieException):
        env.set_observation_delay(0.006)  # more than one 5 ms tick
    env.close()
    plain.close()


# ---- 6. checkpoints and rejections -------------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n, T = 512, 30
    a = _sim(model, _config(), n, 1, sense=(1, 4), delay=(0, 2))
    for k in range(T):
        _step(a, "servos", _action(torch, model, "servos", n, k))
    sd = a.state_dict()
    assert sd["observation_delay"] == (1, 4)
    b = UpkieSim(n, model=model, config=_config())
    b.load_state_dict(sd)
    for k in range(T, 2 * T):
        x = _step(a, "servos", _action(torch, model, "servos", n, k))
        y = _step(b, "servos", _action(torch, model, "servos", n, k))
        for u, v in zip(x, y):
            assert (u is None and v is None) or _bits(u) == _bits(v), k
    for u, v in zip(a.get_observation_delay_state(), b.get_observation_delay_state()):
        assert _bits(u.cpu().numpy()) == _bits(v.cpu().numpy())
    # a checkpoint written before the feature: off, counters 0, delays 0, and nothing allocated on a fresh handle
    old = {k: v for k, v in sd.items() if not k.startswith("observation_delay")}
    c = UpkieSim(n, model=model, config=_config())
    c.load_state_dict(old)
    assert getattr(c, "_observation_delay", None) is None and not getattr(c, "_sense_state_set", False)
    count, delay, rows = (x.cpu().numpy() for x in c.get_observation_delay_state())
    assert not count.any() and not delay.any() and _bits(rows) == _bits(_state(c))
    c.set_observation_delay(2, 3)
    c.load_state_dict(old)
    assert c._observation_delay is None
    count, delay, _ = (x.cpu().numpy() for x in c.get_observation_delay_state())
    assert not count.any() and not delay.any()


def test_rejections_and_none(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 64
    s = UpkieSim(n, model=model, config=_config())
    s.set_observation_delay(1, 2)
    for low, high in ((3, 2), (0, 6)):
        with pytest.raises(UpkieRuntimeError):
            s.set_observation_delay(low, high)
        assert s._observation_delay == (1, 2)
    for cfg in (_config(joint_limits=0), _config(spine_mode=1), _config(body_contacts=1)):
        with pytest.raises(UpkieRuntimeError):
            UpkieSim(n, model=model, config=cfg).set_observation_delay(0, 1)
    # set_config refuses fewer substeps than the range needs, no joint limits and body contacts
    for cfg in (_config(nb_substeps=1), _config(joint_limits=0), _config(body_contacts=1)):
        with pytest.raises(UpkieRuntimeError):
            s.set_config(cfg)
    s.set_config(_config(nb_substeps=2))
    # the in-kernel rollout transports
    m = UpkieSim(64, model=model, config=_config(max_episode_steps=0))
    m.set_observation_delay(0, 1)
    with pytest.raises(UpkieRuntimeError, match="observation delay has no in-kernel rollout transport"):
        obs = torch.empty((64, 18), device="cuda")
        term = torch.empty(64, dtype=torch.uint8, device="cuda")
        m.step_servos_peers(_action(torch, model, "servos", 64, 0), [obs.data_ptr()], [term.data_ptr()])
    # None: the old families and the true state's spine observation
    n, T = 256, 20
    sim = _sim(model, _config(), n, 1, sense=(2, 5), table=True)
    twin = _sim(model, _config(), n, 1, table=True)
    for k in range(5):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    sim.set_observation_delay(None)
    twin.load_state_dict(sim.state_dict())  # same state and counters; the twin never had a spec in force
    for k in range(T):
        x = _step(sim, "servos", _action(torch, model, "servos", n, k))
        y = _step(twin, "servos", _action(torch, model, "servos", n, k))
        for u, v in zip(x, y):
            assert (u is None and v is None) or _bits(u) == _bits(v), k
    # set_state copies the state into the sensed rows while a spec is set
    sim.set_observation_delay(0, 5)
    st = twin.get_state()
    sim.set_state(st)
    torch.cuda.synchronize()
    assert _bits(_rows(sim)) == _bits(st.cpu().numpy())


# ---- 7. reset observations and re-enabling -----------------------------------------------------------------------------


@pytest.mark.parametrize("env_type", ["gyropod", "pendulum"])
def test_masked_reset_returns_the_sensed_observation(torch, env_type):
    # With d = nb_substeps the observation of a step is the state at its start: a masked reset returns, for the envs it
    # does not take, the observation of the last step (their sensed rows are untouched), not one of the true state
    from upkie_b200.envs import B200VectorEnv

    n = 256
    env = B200VectorEnv(n, env_type, autoreset_mode="disabled", observation_delay=0.005)
    assert env.sim._observation_delay == (5, 5)
    env.reset(seed=3)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(11)
    dim = 2 if env_type == "gyropod" else 1
    for _ in range(6):
        obs, _, _, _, _ = env.step_tensors((torch.rand((n, dim), device="cuda", generator=gen) * 2 - 1) * 0.5)
    last = obs.cpu().numpy().copy()
    mask = (np.arange(n) % 3 == 0).astype(np.uint8)
    out, _ = env.reset(options={"reset_mask": mask})
    keep = mask == 0
    # the same sensed state; k_reset_obs is compiled apart from the step kernel, so the orientation-derived columns
    # may round differently in the last bit
    np.testing.assert_allclose(out[keep], last[keep], rtol=1e-6, atol=1e-7)
    # the true state's observation is another: the envs moved during the last tick
    env.set_observation_delay(None)
    plain = env.sim.reset_obs(6 if env_type == "gyropod" else 4).cpu().numpy()
    assert np.abs(plain[keep] - last[keep]).max() > 1e-3
    env.set_observation_delay(0.005)  # turned on again: the rows start from the current state
    assert _bits(env.sim.get_observation_delay_state()[2].cpu().numpy()) == _bits(_state(env.sim))
    env.close()


def test_reset_obs_of_servos_reads_the_sensed_rows(model, torch):
    n, nb = 512, 5
    cfg = _config(max_episode_steps=0, servos_fall_termination=0, nb_substeps=nb)
    sim = _sim(model, cfg, n, 0, sense=(nb, nb))
    sim.set_observation_delay_state(torch.zeros(n, dtype=torch.int32, device="cuda"),
                                    torch.full((n,), nb, dtype=torch.int32, device="cuda"), sim.get_state())
    for k in range(5):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    mask = (np.arange(n) % 2).astype(np.uint8)
    sim.reset(mask=torch.from_numpy(mask).cuda(), seed=SEED)
    obs = sim.reset_obs(_abi.OBS_DIM).cpu().numpy().reshape(n, 6, 5)
    rows, st = _rows(sim), _state(sim)
    for key, col in ((0, _abi.ST_Q), (1, _abi.ST_QD), (2, _abi.ST_TORQUE)):
        assert _bits(obs[:, :, key]) == _bits(rows[:, col:col + 6])
    keep, took = mask == 0, mask == 1
    assert _bits(rows[took]) == _bits(st[took])
    assert not np.array_equal(rows[keep][:, _abi.ST_Q:_abi.ST_Q + 6], st[keep][:, _abi.ST_Q:_abi.ST_Q + 6])


def test_turning_the_delay_on_again_starts_from_the_state(model, torch):
    n = 256
    sim = _sim(model, _config(), n, 1, sense=(2, 5))
    for k in range(8):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    count, delay, _ = (x.cpu().numpy() for x in sim.get_observation_delay_state())
    sim.set_observation_delay(None)
    for k in range(8, 12):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    sim.set_observation_delay(2, 5)
    c2, d2, rows = (x.cpu().numpy() for x in sim.get_observation_delay_state())
    assert _bits(rows) == _bits(_state(sim))  # the rows follow the robot again, IMU velocity included
    assert _bits(c2) == _bits(count) and _bits(d2) == _bits(delay)  # counters and delays stay
    # replacing a spec in force keeps the rows
    _step(sim, "servos", _action(torch, model, "servos", n, 12))
    before = _rows(sim)
    sim.set_observation_delay(1, 5)
    assert _bits(_rows(sim)) == _bits(before)
