# SPDX-License-Identifier: Apache-2.0
"""Servo reply dropouts on the device (upkie_b200_set_servo_dropout): the physics does not depend on the losses, every
servo-derived output reports the triple of the servo's last received reply at the age the NumPy law predicts, the loss
rate, a zero probability against a twin without dropouts on the device and host tiles, same-step terminal
observations, the composition with the observation delay and the history, sharding, checkpoints and the rejections."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_servo_dropout_cpu import SEED as LAW_SEED, lost_np, prob_np

pytestmark = pytest.mark.gpu

SEED = LAW_SEED
SERVO_COLS = [_abi.SP_SERVO + 5 * j + k for j in range(6) for k in range(3)]


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


def _sim(model, cfg, n, mode, drop=None, joints=None, history=True, env_offset=0, sense=None):
    """a handle (FAM_SENSE through a history, so that a twin without dropouts runs the same kernels), reset once"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if history:
        s.set_history([_abi.SP_PITCH, _abi.SP_SERVO, _abi.SP_ODOM_POS], 3)
    if sense is not None:
        s.set_observation_delay(*sense)
    if drop is not None:
        s.set_servo_dropout(drop[0], drop[1], joints)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k, env_offset=0, total=None):
    total = total or n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7000 + k)
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
    """(obs, terminated, truncated, final_obs or None, final spine obs or None, spine obs, history) as NumPy arrays"""
    step = {"servos": sim.step_servos, "gyropod": sim.step_gyropod, "pendulum": sim.step_pendulum}[kind]
    fin = fso = None
    if same_step:
        fin = torch_mod.zeros((sim.n,) + FINAL_SHAPE[kind], device="cuda")
        obs, _, term, trunc = step(a, final_obs=fin, final_state=True)
        fso = sim.final_spine_obs()
    else:
        obs, _, term, trunc = step(a)
    hist = sim.get_history() if sim.history_spec is not None else None
    out = [obs, term, trunc, fin, fso, sim.spine_obs(), hist]
    return [None if x is None else x.clone().cpu().numpy() for x in out]


def _bits(x):
    return np.ascontiguousarray(x).tobytes()


def _state(sim):
    return sim.get_state().cpu().numpy()


def _triples(state):
    """[n, 18] the [joint][q, qd, torque] of state rows"""
    return np.stack([state[:, _abi.ST_Q:_abi.ST_Q + 6], state[:, _abi.ST_QD:_abi.ST_QD + 6],
                     state[:, _abi.ST_TORQUE:_abi.ST_TORQUE + 6]], axis=-1).reshape(-1, 18)


# ---- the physics does not depend on the losses ----------------------------------------------------------------------


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_physics_is_unaffected(model, torch, kind, mode):
    n, T = 256, 200
    cfg = _config()
    sim = _sim(model, cfg, n, mode, drop=(0.2, 0.8))
    twin = _sim(model, cfg, n, mode)
    resets = stale = 0
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        x = _step(sim, kind, a, same_step=mode == 2)
        y = _step(twin, kind, a, same_step=mode == 2)
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
        resets += int((x[1] | x[2]).sum())
        stale += int((x[5][:, SERVO_COLS] != y[5][:, SERVO_COLS]).any(axis=1).sum())
    assert stale > 0 and (mode == 0 or resets > 0)


# ---- zero probability: every output of the twin, bit for bit ----------------------------------------------------------


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["servos", "gyropod"])
def test_zero_probability_matches_the_twin(model, torch, kind, mode):
    n, T = 512, 60
    cfg = _config()
    sim = _sim(model, cfg, n, mode, drop=(0.0, 0.0))
    twin = _sim(model, cfg, n, mode)
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        for x, y in zip(_step(sim, kind, a, same_step=mode == 2), _step(twin, kind, a, same_step=mode == 2)):
            assert (x is None) == (y is None)
            if x is not None:
                assert _bits(x) == _bits(y), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k


def test_zero_probability_host_tiles(model, torch):
    n, T = 512, 40
    cfg = _config()
    sim = _sim(model, cfg, n, 2, drop=(0.0, 0.0))
    twin = _sim(model, cfg, n, 2)
    for k in range(T):
        a = _action(torch, model, "servos", n, k).cpu().numpy().reshape(n, 36)
        x = [np.array(v, copy=True) for v in sim.step_host(a, 36, compact=True, final_obs=True)]
        y = [np.array(v, copy=True) for v in twin.step_host(a, 36, compact=True, final_obs=True)]
        for u, v in zip(x, y):
            assert _bits(u) == _bits(v), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k


# ---- the reported triples are the state at the predicted age ------------------------------------------------------------


def test_reported_values_at_the_predicted_age(model, torch):
    # frequency = 1000: one spine cycle per tick, so a tick's observation is the state at the servo's age in ticks
    n, T, p = 512, 120, 0.3
    cfg = _config(dt=0.001, nb_substeps=1, max_episode_steps=0, servos_fall_termination=0)
    for j in range(6):
        cfg.torque_measurement_noise[j] = 0.0
    mask = 0b110111  # the right hip may not lose replies
    joints = [name for j, name in enumerate(_abi.JOINT_NAMES) if (mask >> j) & 1]
    sim = _sim(model, cfg, n, 0, drop=(p, p), joints=joints, history=False)
    gyro = _sim(model, cfg, n, 0, drop=(p, p), joints=joints, history=False)
    twin = _sim(model, cfg, n, 0, history=False)  # the spine and gyropod observations of a given state
    count, prob, held = sim.get_servo_dropout_state()
    np.testing.assert_array_equal(count.cpu().numpy(), 1)
    np.testing.assert_array_equal(prob.cpu().numpy(), prob_np(p, p, SEED, np.arange(n), 1))
    tick0 = sim.state_dict()["tick"].cpu().numpy().astype(np.uint64)
    truth = [_triples(_state(sim))]  # the explicit reset latched the post-reset state
    gtruth = [_triples(_state(gyro))]
    g = np.arange(n, dtype=np.uint64)
    age = np.zeros((n, 6), dtype=np.int64)
    stale = 0
    for k in range(T):
        obs = sim.step_servos(_action(torch, model, "servos", n, k))[0].cpu().numpy()
        gobs = gyro.step_gyropod(_action(torch, model, "gyropod", n, k))[0].cpu().numpy()
        spine = sim.spine_obs().cpu().numpy()
        state = _state(sim)
        truth.append(_triples(state))
        lost = lost_np(mask, p, SEED, g, tick0 + 1 + k, 0)
        age = np.where(lost, age + 1, 0)
        stale += int(lost.sum())
        src = len(truth) - 1 - age  # [n, 6]
        expect = np.stack([np.stack([truth[src[i, j]][i, 3 * j:3 * j + 3] for j in range(6)]) for i in range(n)])
        assert _bits(obs[:, :, :3]) == _bits(expect), k
        assert _bits(spine[:, SERVO_COLS].reshape(n, 6, 3)) == _bits(expect), k
        # the odometry of the spine observation and the gyropod rows: those of the state with the latched servos
        seen = state.copy()
        for c, col in enumerate((_abi.ST_Q, _abi.ST_QD, _abi.ST_TORQUE)):
            seen[:, col:col + 6] = expect[:, :, c]
        twin.set_state(torch.from_numpy(seen).cuda())
        ref = twin.spine_obs().cpu().numpy()
        assert _bits(spine[:, _abi.SP_ODOM_POS:_abi.SP_ODOM_VEL + 1]) == _bits(ref[:, _abi.SP_ODOM_POS:_abi.SP_ODOM_VEL + 1])
        # the gyropod handle draws the same losses: its rows' ground position and velocity are those of its state with
        # the servos at the same ages (another kernel's arithmetic: fp32 round-off)
        gstate = _state(gyro)
        gtruth.append(_triples(gstate))
        gexp = np.stack([np.stack([gtruth[src[i, j]][i, 3 * j:3 * j + 3] for j in range(6)]) for i in range(n)])
        gseen = gstate.copy()
        for c, col in enumerate((_abi.ST_Q, _abi.ST_QD, _abi.ST_TORQUE)):
            gseen[:, col:col + 6] = gexp[:, :, c]
        twin.set_state(torch.from_numpy(gseen).cuda())
        gref = twin.reset_obs(6).cpu().numpy()
        np.testing.assert_allclose(gobs[:, [0, 3]], gref[:, [0, 3]], rtol=1e-5, atol=1e-5, err_msg=str(k))
    frac = stale / (n * T * 5)  # five servos may lose replies
    assert abs(frac - p) < 5 * np.sqrt(p * (1 - p) / (n * T * 5)), frac


# ---- same-step terminal observations, composition ------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "gyropod"])
def test_same_step_final_observations_report_the_latched_servos(model, torch, kind):
    # p = 1: nothing arrives between resets, so the terminal step reports what the env's last reset latched
    n, T = 512, 40
    cfg = _config(max_episode_steps=7)
    sim = _sim(model, cfg, n, 2, drop=(1.0, 1.0))
    resets = 0
    for k in range(T):
        held = sim.get_servo_dropout_state()[2].cpu().numpy()  # [n, 6, 3]
        out = _step(sim, kind, _action(torch, model, kind, n, k), same_step=True)
        done = (out[1] | out[2]).astype(bool)
        resets += int(done.sum())
        if kind == "servos":
            assert _bits(out[3][done][:, :, :2]) == _bits(held[done][:, :, :2]), k
            assert _bits(out[0][~done][:, :, :2]) == _bits(held[~done][:, :, :2]), k
        fso = out[4][done][:, SERVO_COLS].reshape(-1, 6, 3)
        assert _bits(fso[:, :, :2]) == _bits(held[done][:, :, :2]), k
        # the reset latched the post-reset state
        after = sim.get_servo_dropout_state()[2].cpu().numpy()
        assert _bits(after[done]) == _bits(_triples(_state(sim))[done].reshape(-1, 6, 3)), k
    assert resets > 0


@pytest.mark.parametrize("d", [0, 3, 5])
def test_observation_delay_and_history_take_the_latched_values(model, torch, d):
    n, T = 256, 12
    cfg = _config(max_episode_steps=0, servos_fall_termination=0)
    sim = _sim(model, cfg, n, 0, drop=(1.0, 1.0), sense=(d, d))
    held = sim.get_servo_dropout_state()[2].cpu().numpy()
    assert _bits(held) == _bits(_triples(_state(sim)).reshape(n, 6, 3))
    for k in range(T):
        out = _step(sim, "servos", _action(torch, model, "servos", n, k))
        assert _bits(out[0][:, :, :2]) == _bits(held[:, :, :2]), k
        assert _bits(out[5][:, SERVO_COLS].reshape(n, 6, 3)[:, :, :2]) == _bits(held[:, :, :2]), k
        # the history's servo column (left hip position) in every entry
        assert (out[6][:, :, 1] == held[:, None, 0, 0]).all(), k
        assert _bits(sim.get_servo_dropout_state()[2].cpu().numpy()) == _bits(held), k


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 40
    whole = _sim(model, _config(), n, 2, drop=(0.1, 0.6))
    half = n // 2
    shards = [_sim(model, _config(), half, 2, drop=(0.1, 0.6), env_offset=o) for o in (0, half)]
    for k in range(T):
        out = _step(whole, "servos", _action(torch, model, "servos", n, k))
        for s, o in zip(shards, (0, half)):
            part = _step(s, "servos", _action(torch, model, "servos", half, k, env_offset=o, total=n))
            assert _bits(part[0]) == _bits(out[0][o : o + half]), k
            assert _bits(part[5]) == _bits(out[5][o : o + half]), k
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_servo_dropout_state(), whole.get_servo_dropout_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o : o + half])


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 256
    cfg = _config()
    sim = _sim(model, cfg, n, 2, drop=(0.2, 0.5), joints=["left_wheel", "right_wheel"])
    for k in range(10):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    sd = sim.state_dict()
    assert sd["servo_dropout"][2] == (1 << 2) | (1 << 5)
    ref = [_step(sim, "servos", _action(torch, model, "servos", n, 10 + k)) for k in range(10)]
    other = UpkieSim(n, model=model, config=cfg)
    other.load_state_dict(sd)
    for k in range(10):
        for x, y in zip(_step(other, "servos", _action(torch, model, "servos", n, 10 + k)), ref[k]):
            if x is not None:
                assert _bits(x) == _bits(y), k
    # a checkpoint without dropouts turns them off
    del sd["servo_dropout"]
    other.load_state_dict(sd)
    assert other.servo_dropout_spec is None


def test_rejections_and_none(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 64
    sim = _sim(model, _config(), n, 1, drop=(0.1, 0.2), history=False)
    for bad in ((0.3, 0.2), (-0.1, 0.2), (0.0, 1.5)):
        with pytest.raises((UpkieException, UpkieRuntimeError), match="prob_low"):
            sim.set_servo_dropout(*bad)
    with pytest.raises(UpkieException, match="unknown joint"):
        sim.set_servo_dropout(0.1, 0.2, ["left_elbow"])
    assert sim.servo_dropout_spec[:2] == (np.float32(0.1), np.float32(0.2))  # the previous spec is kept
    for field, value, what in (("joint_limits", 0, "joint_limits"), ("body_contacts", 1, "body_contacts")):
        cfg = _config(**{field: value})
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_config(cfg)
    spine = UpkieSim(n, model=model, config=_config(spine_mode=1))
    with pytest.raises((UpkieException, UpkieRuntimeError), match="spine_mode"):
        spine.set_servo_dropout(0.1)
    sim.set_servo_dropout(None)
    assert sim.servo_dropout_spec is None
    with pytest.raises(UpkieException, match="no servo dropouts"):
        sim.get_servo_dropout_state()
    sim.step_servos(_action(torch, model, "servos", n, 0))


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200.envs import B200VectorEnv

    env = B200VectorEnv(64, env_type=env_type, autoreset_mode="next_step", servo_dropout=(0.1, 0.3),
                        servo_dropout_joints=["left_wheel", "right_wheel"])
    env.reset(seed=3)
    count, prob, _ = env.sim.get_servo_dropout_state()
    assert (count.cpu().numpy() == 1).all()
    np.testing.assert_array_equal(prob.cpu().numpy(), prob_np(0.1, 0.3, 3, np.arange(64), 1))
    for _ in range(5):
        env.step(env.action_space.sample())
    env.set_servo_dropout(None)
    env.step(env.action_space.sample())
    with pytest.raises(UpkieException, match="servo_dropout"):
        B200VectorEnv(8, env_type=env_type, servo_dropout=(0.5, 0.2))


# ---- mid-tick instants: several cycles per tick, 0 < p < 1 ------------------------------------------------------------


@pytest.mark.parametrize("d", [0, 2])
def test_mid_tick_instants_at_the_predicted_age(model, torch, d):
    # nb = 5 cycles per tick: the history's entries and the observation (under an observation delay of d substeps, the
    # snapshot nb - 1 - d substeps into the tick) report each servo at the age the NumPy law predicts. A twin without
    # dropouts and with the same history and delay records the true values of the same instants.
    n, T, p, nb, K = 256, 30, 0.4, 5, 5
    cfg = _config(nb_substeps=nb, max_episode_steps=0, servos_fall_termination=0)
    cols = [_abi.SP_SERVO + 5 * j + k for j in range(6) for k in range(2)]  # positions and velocities
    sims = []
    for drop in ((p, p), None):
        s = _sim(model, cfg, n, 0, drop=drop, history=False, sense=(d, d))
        s.set_history(cols, K)
        sims.append(s)
    sim, twin = sims
    tick0 = sim.state_dict()["tick"].cpu().numpy().astype(np.uint64)
    init = _triples(_state(sim)).reshape(n, 6, 3)[:, :, :2].reshape(n, 12)  # the latch of the explicit reset
    truth = {}  # global substep index t * nb + s -> [n, 12] true values after it
    g = np.arange(n, dtype=np.uint64)
    age = np.zeros((n, 6), dtype=np.int64)
    ages = {}
    stale = 0
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        obs = sim.step_servos(a)[0].cpu().numpy()
        twin.step_servos(a)
        hs, ht = sim.get_history().cpu().numpy(), twin.get_history().cpu().numpy()
        for s in range(nb):
            lost = lost_np(0x3F, p, SEED, g, tick0 + 1 + k, s)
            age = np.where(lost, age + 1, 0)
            ages[k * nb + s] = age.copy()
            stale += int(lost.sum())
        for e in range(K):
            G = k * nb + nb - 1 - d - e
            if G >= 0:
                truth.setdefault(G, ht[:, e])
        for e in range(K):
            G = k * nb + nb - 1 - d - e
            if G < 0:
                continue
            src = G - ages[G]  # [n, 6]
            expect = np.empty((n, 12), dtype=np.float32)
            for j in range(6):
                for i in range(n):
                    v = truth[src[i, j]] if src[i, j] >= 0 else init
                    expect[i, 2 * j:2 * j + 2] = v[i, 2 * j:2 * j + 2]
            assert _bits(hs[:, e]) == _bits(expect), (k, e)
            if e == 0:  # the observation reports the history's newest entry
                assert _bits(obs[:, :, :2].reshape(n, 12)) == _bits(expect), k
    assert stale > 0


def test_a_wider_mask_latches_the_added_servos(model, torch):
    # the wheels only, then every servo at p = 0: the legs' held rows follow the state from the new spec on
    n, T = 256, 20
    cfg = _config()
    sim = _sim(model, cfg, n, 1, drop=(0.0, 0.0), joints=["left_wheel", "right_wheel"])
    twin = _sim(model, cfg, n, 1)
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        if k == T // 2:
            sim.set_servo_dropout(0.0, 0.0)
            assert _bits(sim.spine_obs().cpu().numpy()) == _bits(twin.spine_obs().cpu().numpy())
        for x, y in zip(_step(sim, "servos", a), _step(twin, "servos", a)):
            if x is not None:
                assert _bits(x) == _bits(y), k
