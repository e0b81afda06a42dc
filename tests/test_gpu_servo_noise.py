# SPDX-License-Identifier: Apache-2.0
"""Servo measurement noise on the device (upkie_b200_set_servo_noise): the physics and torques of an UpkieServos handle
with noise are a twin's without it; the residuals are the drawn sigmas times standard normals; one cycle reports one
value in every output; an observation delay of d substeps reports history entry d of an undelayed twin; a lost reply
repeats the noisy reply it last received; encoder offsets add to the noisy reply; reset observations and the leg
targets they set carry the reset cycle's noise; zero ranges and NULL are a handle without the feature; checkpoints and
reseeded resets repeat runs; the vector envs, base velocity included."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, _abi
from test_servo_noise_cpu import sigma_np, make_spec

pytestmark = pytest.mark.gpu

SEED = 0x5E12C0
NEXT_STEP, SAME_STEP = 1, 2
LEGS = [0, 1, 3, 4]
LT = slice(_abi.ST_LEG_TARGET, _abi.ST_LEG_TARGET + 4)
POS = [_abi.SP_SERVO + j * 5 for j in range(6)]  # the servo positions of a spine row
VEL = [p + 1 for p in POS]
# history columns: every servo position and velocity, the odometry, the pitch
HISTORY = POS + VEL + [_abi.SP_ODOM_POS, _abi.SP_ODOM_VEL, _abi.SP_PITCH]
FINAL_SHAPE = {"servos": (6, 5), "gyropod": (6,), "pendulum": (4,)}
# position noise on every joint but the left knee, velocity noise on every joint but the right knee
P_HI = np.array([0.01, 0.0, 0.01, 0.01, 0.01, 0.01], np.float32)
V_HI = np.array([0.5, 0.5, 0.5, 0.5, 0.0, 0.5], np.float32)


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


def _sim(model, cfg, n, mode, noise=True, history=HISTORY, size=5, sense=None, drop=(0.0, 0.0), offset=None,
         max_ticks=1):
    """a handle reset once; a zero-probability servo-dropout spec runs it in FAM_SENSE, so that a twin without the
    noise runs the same kernels"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, 0)
    if history:
        s.set_history(history, size)
    if sense is not None:
        s.set_observation_delay(sense, sense, max_ticks=max_ticks)
    if drop is not None:
        s.set_servo_dropout(*drop)
    if offset is not None:
        s.set_encoder_offset(-offset, offset, list(_abi.JOINT_NAMES))
    if noise is True:
        s.set_servo_noise((np.zeros(6), P_HI), (np.zeros(6), V_HI))
    elif noise is not None:
        s.set_servo_noise(*noise)
    s.reset(seed=SEED)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k, shift=None):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7000 + k)
    if kind == "servos":
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 4.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
        if shift is not None:
            a[:, :, 0] -= torch.from_numpy(shift).cuda()
        return a
    dim = 2 if kind == "gyropod" else 1
    return ((torch.rand((n, dim), device="cuda", generator=gen) * 2 - 1) * 2.0).contiguous()


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


def _same_state(a, b):
    """get_state bit for bit, the leg targets aside (a reset sets them from its noisy observation, an UpkieServos
    handle's too, unused)"""
    other = np.ones(_abi.STATE_DIM, bool)
    other[LT] = False
    return _bits(_state(a)[:, other]) == _bits(_state(b)[:, other])


def _sigma(sim):
    return sim.get_servo_noise_state()[1].cpu().numpy()


# ---- 1, 2. the physics is the twin's; the residuals are sigma times standard normals -----------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_servos_twin_and_residual_statistics(model, torch, mode):
    n, T = 512, 200
    sim = _sim(model, _config(), n, mode)
    twin = _sim(model, _config(), n, mode, noise=None)
    same = mode == SAME_STEP
    z = [[] for _ in range(12)]
    zero_cols = 0
    resets = 0
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        x = _step(sim, "servos", a, same)
        y = _step(twin, "servos", a, same)
        st, tt = _state(sim), _state(twin)
        other = np.ones(_abi.STATE_DIM, bool)
        other[LT] = False
        assert _bits(st[:, other]) == _bits(tt[:, other]), k  # get_state bit for bit (UpkieServos leg targets aside)
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        assert _bits(x[0][:, :, 2:]) == _bits(y[0][:, :, 2:]), k  # torques, temperature, voltage
        sg = _sigma(sim)
        for q in range(2):
            res = (x[0][:, :, q] - y[0][:, :, q]).astype(np.float64)
            for j in range(6):
                s = sg[:, 6 * q + j]
                if (P_HI if q == 0 else V_HI)[j] == 0:
                    assert (res[:, j] == 0).all(), (k, q, j)  # a zero range: exactly the twin's
                    zero_cols += 1
                    continue
                ok = s > (1e-3 if q == 0 else 0.05)
                z[6 * q + j].append(res[ok, j] / s[ok])
        resets += int((x[1] | x[2]).sum())
    assert resets > n and zero_cols == 2 * T
    for c in range(12):
        if not z[c]:
            continue
        v = np.concatenate(z[c])
        assert len(v) > 50000
        assert abs(v.mean()) < 0.03, (c, v.mean())
        assert abs(v.std() - 1.0) < 0.03, (c, v.std())
    # the drawn sigmas follow the law of the header: draw `count` of every env
    count, sg = sim.get_servo_noise_state()
    spec = make_spec(0.0, P_HI, 0.0, V_HI)
    np.testing.assert_array_equal(sg.cpu().numpy(), np.concatenate(
        [sigma_np(spec, SEED, [i], int(c)) for i, c in enumerate(count.cpu().numpy().astype(np.uint32))]))


# ---- 3. one cycle, one value --------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_one_cycle_one_value(model, torch, mode):
    n, T = 256, 80
    sim = _sim(model, _config(), n, mode)
    twin = _sim(model, _config(), n, mode, noise=None)
    same = mode == SAME_STEP
    finals = 0
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        x = _step(sim, "servos", a, same)
        y = _step(twin, "servos", a, same)
        obs, sp, h = x[0], x[5], x[6]
        # the step row, spine_obs and history entry 0, resets included
        assert _bits(obs[:, :, 0]) == _bits(sp[:, POS]) == _bits(h[:, 0, 0:6]), k
        assert _bits(obs[:, :, 1]) == _bits(sp[:, VEL]) == _bits(h[:, 0, 6:12]), k
        np.testing.assert_allclose(h[:, 0, 12:14], sp[:, [_abi.SP_ODOM_POS, _abi.SP_ODOM_VEL]], atol=1e-6)
        # distinct entries carry distinct noise (the twin's entries are the same substeps without it)
        res = h[:, :, :12] - y[6][:, :, :12]
        live = _sigma(sim)[:, 0] > 1e-3
        for e in range(1, h.shape[1]):
            assert (res[live, e, 0] != res[live, 0, 0]).mean() > 0.99, (k, e)
        done = (x[1] | x[2]).astype(bool)
        if same and done.any():
            fin, fso = x[3][done], x[4][done]
            assert _bits(fin[:, :, 0]) == _bits(fso[:, POS]) and _bits(fin[:, :, 1]) == _bits(fso[:, VEL]), k
            assert _bits(fin[:, :, 2:]) == _bits(y[3][done][:, :, 2:]), k
            finals += int(done.sum())
    assert finals > 0 or not same


# ---- 4. an observation delay of d substeps is history entry d --------------------------------------------------------


@pytest.mark.parametrize("d,max_ticks", [(3, 1), (5, 1), (8, 2)])
def test_delay_is_history_entry_d(model, torch, d, max_ticks):
    n, T = 256, 60
    delayed = _sim(model, _config(), n, NEXT_STEP, history=None, sense=d, max_ticks=max_ticks, drop=None)
    plain = _sim(model, _config(), n, NEXT_STEP, size=12, drop=None)
    # the reset before tick 0 counts: right after a reset, the newest entry of a refilled history is the reset
    # observation, while a delayed snapshot of the refilled rows is reported with the noise of the cycle it stands for
    reset_at = np.zeros(n, dtype=np.int64)
    checked = 0
    done_prev = np.zeros(n, bool)
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        x = _step(delayed, "servos", a)
        y = _step(plain, "servos", a)
        assert _bits(_state(delayed)) == _bits(_state(plain)), k
        reset_at[done_prev] = k
        ok = k - reset_at > 2  # no reset in the window the delay reaches back into
        np.testing.assert_array_equal(x[0][ok, :, 0], y[6][ok, d, 0:6], err_msg=str(k))
        np.testing.assert_array_equal(x[0][ok, :, 1], y[6][ok, d, 6:12], err_msg=str(k))
        # spine_obs reports the same delayed cycle
        np.testing.assert_array_equal(x[5][ok][:, POS], y[6][ok, d, 0:6], err_msg=str(k))
        checked += int(ok.sum())
        done_prev = (x[1] | x[2]).astype(bool)
    assert checked > n * T // 2


# ---- 5. a lost reply repeats the noisy reply last received ----------------------------------------------------------


def test_dropouts_hold_the_noisy_reply(model, torch):
    n, T = 256, 120
    sim = _sim(model, _config(max_episode_steps=0), n, NEXT_STEP, drop=(0.5, 0.5))
    twin = _sim(model, _config(max_episode_steps=0), n, NEXT_STEP, noise=None, drop=(0.5, 0.5))
    prev = prev_twin = None
    held = 0
    done_prev = np.zeros(n, bool)
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        x = _step(sim, "servos", a)
        y = _step(twin, "servos", a)
        assert _same_state(sim, twin), k
        if prev is not None:
            # the twin's servo kept its reply of the last tick (every cycle of this one lost it): so does the noisy one
            same = (y[0][:, :, 0] == prev_twin[:, :, 0]) & (y[0][:, :, 1] == prev_twin[:, :, 1])
            same &= ~done_prev[:, None]
            assert _bits(x[0][:, :, :2][same]) == _bits(prev[:, :, :2][same]), k
            held += int(same.sum())
            # a servo received in this tick reports the twin's reply plus noise
            moved = ~same & ~done_prev[:, None]
            assert (x[0][:, :, 0][moved & (P_HI > 0)] != y[0][:, :, 0][moved & (P_HI > 0)]).mean() > 0.99
        prev, prev_twin = x[0], y[0]
        done_prev = (x[1] | x[2]).astype(bool)
    assert held > 1000


# ---- 6. encoder offsets: q + noise + delta --------------------------------------------------------------------------


def test_encoder_offsets_add_to_the_noisy_reply(model, torch):
    n, T = 256, 60
    sim = _sim(model, _config(), n, SAME_STEP, offset=0.05)
    twin = _sim(model, _config(), n, SAME_STEP)
    for k in range(T):
        d_old = sim.get_encoder_offset_state()[1].cpu().numpy()
        x = _step(sim, "servos", _action(torch, model, "servos", n, k), True)
        y = _step(twin, "servos", _action(torch, model, "servos", n, k, shift=d_old), True)
        d = sim.get_encoder_offset_state()[1].cpu().numpy()
        assert _bits(x[1]) == _bits(y[1]), k
        np.testing.assert_array_equal(x[0][:, :, 0], y[0][:, :, 0] + d, err_msg=str(k))
        assert _bits(x[0][:, :, 1]) == _bits(y[0][:, :, 1]), k
        np.testing.assert_array_equal(x[5][:, POS], y[5][:, POS] + d, err_msg=str(k))


# ---- 7. reset observations ----------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["gyropod", "pendulum"])
def test_reset_observation_and_leg_targets(model, torch, kind):
    n = 256
    sim = _sim(model, _config(), n, SAME_STEP)
    twin = _sim(model, _config(), n, SAME_STEP, noise=None)
    # an explicit reset: the leg targets are the reset observation's reported hip and knee positions
    sp = sim.spine_obs().cpu().numpy()
    np.testing.assert_array_equal(_state(sim)[:, LT], sp[:, [POS[j] for j in LEGS]])
    assert (_state(sim)[:, LT] != _state(twin)[:, LT]).mean() > 0.7  # (no position noise on the left knee)
    seen = 0
    for k in range(60):
        x = _step(sim, kind, _action(torch, model, kind, n, k), True)
        y = _step(twin, kind, _action(torch, model, kind, n, k), True)
        done = (x[1] | x[2]).astype(bool)
        # a fused reset: the same, for the envs that reset
        np.testing.assert_array_equal(_state(sim)[done][:, LT], x[5][done][:, [POS[j] for j in LEGS]])
        seen += int(done.sum())
        last, last_twin, last_sigma = x[5], y[5], _sigma(sim)
    assert seen > 0
    # the reset observation's noise is not the preceding step's
    sim.reset(seed=SEED + 1)
    twin.reset(seed=SEED + 1)
    r, rt = sim.spine_obs().cpu().numpy(), twin.spine_obs().cpu().numpy()
    s_new = _sigma(sim)
    ok = (last_sigma[:, 0] > 1e-3) & (s_new[:, 0] > 1e-3)
    z_step = (last[ok, POS[0]] - last_twin[ok, POS[0]]) / last_sigma[ok, 0]
    z_reset = (r[ok, POS[0]] - rt[ok, POS[0]]) / s_new[ok, 0]
    assert (np.abs(z_step - z_reset) > 1e-3).mean() > 0.95
    # reset_obs reports the same reset cycle as spine_obs, bit for bit: the wheel odometry and its rate
    obs6 = sim.reset_obs(6 if kind == "gyropod" else 4).cpu().numpy()
    ro = twin.reset_obs(6 if kind == "gyropod" else 4).cpu().numpy()
    p, pdot = (0, 3) if kind == "gyropod" else (1, 3)  # gyropod [p, pitch, yaw, pdot, ...], pendulum [pitch, p, ., pdot]
    assert _bits(obs6[:, p]) == _bits(r[:, _abi.SP_ODOM_POS])
    assert _bits(obs6[:, pdot]) == _bits(r[:, _abi.SP_ODOM_VEL])
    assert (obs6[:, p] != ro[:, p]).mean() > 0.9


# ---- 8. zero ranges and NULL --------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_zero_ranges_and_null_change_nothing(model, torch, kind, mode):
    n, T = 256, 80
    zero = ((np.zeros(6), np.zeros(6)), (np.zeros(6), np.zeros(6)))
    sim = _sim(model, _config(), n, mode, noise=zero)
    off = _sim(model, _config(), n, mode)  # noise switched off after its first draws
    twin = _sim(model, _config(), n, mode, noise=None)
    off.set_servo_noise(None)
    assert off.servo_noise_spec is None
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        x = _step(sim, kind, a, mode == SAME_STEP)
        y = _step(twin, kind, a, mode == SAME_STEP)
        z = _step(off, kind, a, mode == SAME_STEP)
        for u, v, w in zip(x, y, z):
            if u is not None:
                assert _bits(u) == _bits(v), k
                if kind == "servos":  # (the gyropod and pendulum legs hold targets set with the reset's noise)
                    assert _bits(w) == _bits(v), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
    assert (_sigma(sim) == 0).all()


# ---- 9. checkpoints and seeds -------------------------------------------------------------------------------------------


def test_state_dict_round_trip_and_same_seeds(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 128
    a_sim = _sim(model, _config(), n, SAME_STEP)
    b_sim = _sim(model, _config(), n, SAME_STEP)
    for k in range(30):
        a = _action(torch, model, "servos", n, k)
        x, y = _step(a_sim, "servos", a, True), _step(b_sim, "servos", a, True)
        for u, v in zip(x, y):
            assert _bits(u) == _bits(v), k
    sd = a_sim.state_dict()
    assert "servo_noise" in sd and sd["servo_noise_sigma"].shape == (n, 12)
    c_sim = UpkieSim(n, model=model, config=_config())
    c_sim.load_state_dict(sd)
    for k in range(30, 60):
        a = _action(torch, model, "servos", n, k)
        x, z = _step(a_sim, "servos", a, True), _step(c_sim, "servos", a, True)
        for u, v in zip(x, z):
            assert _bits(u) == _bits(v), k
    # an older checkpoint loads with the feature off
    old = {k: v for k, v in sd.items() if not k.startswith("servo_noise")}
    c_sim.load_state_dict(old)
    assert c_sim.servo_noise_spec is None


def test_vector_env_seeds_restart_the_draws(torch):
    from upkie_b200.envs import B200VectorEnv

    noise = {"position": (0.0, 0.01), "velocity": (0.0, 0.5)}
    envs = [B200VectorEnv(64, "servos", servo_noise=noise) for _ in range(2)]
    envs[0].action_space.seed(3)
    acts = [envs[0].action_space.sample() for _ in range(10)]
    runs = []
    for env in envs:  # two envs with the same seeds: the same runs
        env.reset(seed=11)
        out = [env.sim.spine_obs().cpu().numpy()]
        for a in acts:
            env.step(a)
            out.append(env.sim.spine_obs().cpu().numpy())
        runs.append(out)
    for u, v in zip(*runs):
        assert _bits(u) == _bits(v)
    # reset(seed=s) restarts the draw counters: the same levels as the first reset with that seed
    env = envs[0]
    env.reset(seed=11)
    c1, s1 = (x.cpu().numpy() for x in env.sim.get_servo_noise_state())
    for _ in range(5):
        env.step(env.action_space.sample())
    env.reset(seed=11)
    c2, s2 = (x.cpu().numpy() for x in env.sim.get_servo_noise_state())
    assert (c1 == 1).all() and _bits(c1) == _bits(c2) and _bits(s1) == _bits(s2)
    env.reset(seed=12)
    assert _bits(env.sim.get_servo_noise_state()[1].cpu().numpy()) != _bits(s1)
    for e in envs:
        e.close()


# ---- 10. the vector envs ------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("autoreset", ["disabled", "next_step", "same_step"])
def test_base_velocity_runs_under_noise(torch, autoreset):
    from upkie_b200.envs import B200VectorEnv

    env = B200VectorEnv(64, "base_velocity", autoreset_mode=autoreset,
                        servo_noise={"position": 0.002, "velocity": {"left_wheel": (0.0, 1.0), "right_wheel": 0.5}})
    assert env.sim.servo_noise_spec is not None
    obs, _ = env.reset(seed=5)
    for k in range(40):
        a = env.action_space.sample()
        obs, rew, term, trunc, info = env.step(a)
        assert np.isfinite(np.asarray(obs)).all(), k
    env.close()


@pytest.mark.parametrize("env_id", ["Upkie-B200-Servos", "Upkie-B200-Gyropod", "Upkie-B200-Pendulum",
                                    "Upkie-B200-BaseVelocity"])
def test_make_vec_and_rejections(torch, env_id):
    import upkie_b200

    env = upkie_b200.make_vec(env_id, 16, servo_noise={"velocity": 0.1})
    env.reset(seed=1)
    c, s = env.sim.get_servo_noise_state()
    assert (c.cpu().numpy() == 1).all() and (s.cpu().numpy()[:, 6:] == np.float32(0.1)).all()
    assert (s.cpu().numpy()[:, :6] == 0).all()
    env.step(env.action_space.sample())
    env.set_servo_noise(None)
    assert env.sim.servo_noise_spec is None
    env.close()
    with pytest.raises(UpkieException, match="servo_noise"):
        upkie_b200.make_vec(env_id, 4, servo_noise={"velocity": {"left_elbow": 0.1}})


def test_device_rejections(model, torch):
    from upkie_b200 import UpkieRuntimeError

    n = 32
    sim = _sim(model, _config(), n, NEXT_STEP, history=None)
    good = sim.get_servo_noise_state()
    for bad in (((np.zeros(6), np.full(6, 0.2)), None), ((np.full(6, -0.1), np.zeros(6)), None),
                (None, (np.zeros(6), np.full(6, np.nan)))):
        with pytest.raises((UpkieException, UpkieRuntimeError)):
            sim.set_servo_noise(*bad)
    assert sim.servo_noise_spec is not None  # the previous spec is kept
    c, s = good
    for v in (np.nan, -0.001, 0.11):
        t = s.clone()
        t[0, 0] = float(v)
        with pytest.raises((UpkieException, UpkieRuntimeError)):
            sim.set_servo_noise_state(c, t)
    t = s.clone()
    t[0, 1] = 0.001  # the left knee's position range is zero
    with pytest.raises((UpkieException, UpkieRuntimeError)):
        sim.set_servo_noise_state(c, t)
    sim.set_servo_noise_state(c, s)
    # an observation delay with dropouts and noise: the third is refused
    with pytest.raises((UpkieException, UpkieRuntimeError)):
        sim.set_observation_delay(2, 2)
    cfg = _config()
    cfg.joint_limits = 0
    with pytest.raises((UpkieException, UpkieRuntimeError)):
        sim.set_config(cfg)


# ---- every reset is a cycle of its own; narrowed ranges; checkpoints around resets ----------------------------------


def test_host_row_resets_report_new_normals(model, torch):
    """resets from host rows count no episode; each still reports the normals of its own draw"""
    n = 256
    sim = _sim(model, _config(), n, NEXT_STEP, history=None)
    twin = _sim(model, _config(), n, NEXT_STEP, noise=None, history=None)
    rows = torch.zeros((n, _abi.INIT_DIM), device="cuda")
    rows[:, _abi.INIT_POS + 2] = 0.6
    rows[:, _abi.INIT_QUAT] = 1.0
    rows[:, _abi.INIT_Q:_abi.INIT_Q + 6] = 0.1
    z = []
    for _ in range(3):
        sim.reset(init_state=rows, seed=SEED)
        twin.reset(init_state=rows, seed=SEED)
        a, b, sg = sim.spine_obs().cpu().numpy(), twin.spine_obs().cpu().numpy(), _sigma(sim)
        ok = sg[:, 0] > 1e-3
        z.append(np.where(ok, (a[:, POS[0]] - b[:, POS[0]]) / np.where(ok, sg[:, 0], 1), np.nan))
        # the reset observation: reset_obs, spine_obs and the leg targets agree
        ro = sim.reset_obs(30).cpu().numpy()
        assert _bits(ro[:, :, 0]) == _bits(a[:, POS]) and _bits(ro[:, :, 1]) == _bits(a[:, VEL])
        np.testing.assert_array_equal(_state(sim)[:, LT], a[:, [POS[j] for j in LEGS]])
    for u, v in ((z[0], z[1]), (z[1], z[2])):
        ok = np.isfinite(u) & np.isfinite(v)
        assert ok.sum() > n // 4 and (np.abs(u[ok] - v[ok]) > 1e-3).mean() > 0.95
    # so in a vector env, whose resets take host rows: two resets without a seed, then one with the first's seed
    from upkie_b200.envs import B200VectorEnv

    env = B200VectorEnv(64, "gyropod", servo_noise={"position": (0.0, 0.01), "velocity": (0.0, 0.5)})
    env.reset(seed=4)
    first = env.sim.spine_obs().cpu().numpy()[:, POS + VEL]
    env.reset()
    assert (env.sim.spine_obs().cpu().numpy()[:, POS[0]] != first[:, 0]).mean() > 0.9
    env.reset(seed=4)  # the counters restart: the first reset's draws and normals again
    assert _bits(env.sim.spine_obs().cpu().numpy()[:, POS + VEL]) == _bits(first)
    env.close()


def test_narrowed_range_keeps_round_trips(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import UpkieSim

    env = B200VectorEnv(64, "servos", autoreset_mode="next_step",
                        servo_noise={"position": (0.0, 0.01), "velocity": (0.0, 0.5)})
    env.reset(seed=2)
    env.set_servo_noise({"position": (0.0, 0.005), "velocity": (0.0, 0.1)})  # at each env's next reset
    sg = env.sim.get_servo_noise_state()[1].cpu().numpy()
    assert (sg[:, 0] > 0.005).any() and (sg[:, 6:] > 0.1).any()  # the old levels, above the new bounds
    sd = env.sim.state_dict()
    other = UpkieSim(64, model=env.sim.model, config=env.config)
    other.load_state_dict(sd)
    for k in range(3):
        a = _action(torch, model, "servos", 64, k)
        x, y = _step(env.sim, "servos", a), _step(other, "servos", a)
        for u, v in zip(x, y):
            if u is not None:
                assert _bits(u) == _bits(v), k
    env.reset(seed=2)  # restarts the counters through a state round trip, then draws within the new ranges
    sg = env.sim.get_servo_noise_state()[1].cpu().numpy()
    assert (sg[:, :6] <= np.float32(0.005)).all() and (sg[:, 6:] <= np.float32(0.1)).all()
    env.close()


@pytest.mark.parametrize("kind", ["servos", "gyropod"])
def test_checkpoint_right_after_a_reset(model, torch, kind):
    from upkie_b200.sim import UpkieSim

    n = 64
    sim = _sim(model, _config(), n, SAME_STEP)
    for k in range(5):
        _step(sim, kind, _action(torch, model, kind, n, k), True)
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::2] = 1
    sim.reset(mask=mask, seed=SEED + 3)  # half the envs report their reset observation, half their last step's
    mark = sim.get_servo_noise_mark().cpu().numpy()
    assert (mark[::2] == 1).all() and (mark[1::2] == 0).all()
    sd = sim.state_dict()
    other = UpkieSim(n, model=model, config=_config())
    other.load_state_dict(sd)
    assert _bits(other.spine_obs().cpu().numpy()) == _bits(sim.spine_obs().cpu().numpy())
    dim = 30 if kind == "servos" else 6
    assert _bits(other.reset_obs(dim).cpu().numpy()) == _bits(sim.reset_obs(dim).cpu().numpy())
    for k in range(5, 10):
        a = _action(torch, model, kind, n, k)
        x, y = _step(sim, kind, a, True), _step(other, kind, a, True)
        for u, v in zip(x, y):
            assert _bits(u) == _bits(v), k


def test_load_order_with_delay_and_dropouts(model, torch):
    """a handle with noise and dropouts loads a checkpoint with a delay and dropouts and no noise, and back"""
    from upkie_b200.sim import UpkieSim

    n = 32
    plain = _sim(model, _config(), n, NEXT_STEP, noise=None, sense=2, drop=(0.2, 0.2))
    noisy = _sim(model, _config(), n, NEXT_STEP, drop=(0.2, 0.2))
    sd_plain, sd_noisy = plain.state_dict(), noisy.state_dict()
    noisy.load_state_dict(sd_plain)
    assert noisy.servo_noise_spec is None
    a = _action(torch, model, "servos", n, 0)
    for u, v in zip(_step(noisy, "servos", a), _step(plain, "servos", a)):
        if u is not None:
            assert _bits(u) == _bits(v)
    other = UpkieSim(n, model=model, config=_config())
    other.load_state_dict(sd_plain)
    other.load_state_dict(sd_noisy)
    assert other.servo_noise_spec is not None and getattr(other, "_observation_delay", None) is None
