# SPDX-License-Identifier: Apache-2.0
"""Servo torque scales on the device (upkie_b200_set_torque_scale): a unit scale changes nothing, alone and with the
action delay, servo noise, encoder offsets, velocity limits and a history; a handle with drawn scales matches, bit for
bit, a twin without them that is fed the scaled feedforward torque, while the torque replies keep the command; the
draws follow the NumPy law over fused, explicit, masked, host-row, sharded and chunked host-buffer resets; checkpoints
and fixed scales; the rejections, None and replacement; the vector envs."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_torque_scale_cpu import TAU_MAX, make_spec, scales_np

pytestmark = pytest.mark.gpu

SEED = 0x75CA1E
NEXT_STEP, SAME_STEP = 1, 2
ALL = list(_abi.JOINT_NAMES)
WHEELS = ["left_wheel", "right_wheel"]
FINAL_SHAPE = {"servos": (6, 5), "gyropod": (6,), "pendulum": (4,)}
HISTORY = [_abi.SP_SERVO + 1, _abi.SP_SERVO + 2, _abi.SP_ODOM_VEL, _abi.SP_PITCH]  # a velocity and a torque reply
TORQUE_COLS = list(range(_abi.ST_TORQUE, _abi.ST_TORQUE + 6))
OTHER_COLS = [c for c in range(_abi.STATE_DIM) if c not in TORQUE_COLS]


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


def _sim(model, cfg, n, mode, scale=None, joints=ALL, drop=(0.0, 0.0), env_offset=0, extras=False):
    """a handle reset once; a zero-probability servo-dropout spec runs it in FAM_SENSE, so that a twin without the
    scales runs the same kernels. `extras`: the action delay, servo noise, encoder offsets, velocity limits (that
    bind) and a history on too"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if drop is not None:
        s.set_servo_dropout(*drop)
    if extras:
        s.set_history(HISTORY, 3)
        s.set_action_delay(1, 4)
        s.set_encoder_offset(-0.05, 0.05, ALL)
        s.set_servo_noise((np.zeros(6), np.full(6, 0.005)), (np.zeros(6), np.full(6, 0.3)))
        s.set_velocity_derate((4.0, 12.0), 3.0, ALL)
    if scale is not None:
        s.set_torque_scale(scale, joints)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(7000 + k)
    if kind == "servos":
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 20.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
        return a
    dim = 2 if kind == "gyropod" else 1
    return ((torch.rand((n, dim), device="cuda", generator=gen) * 2 - 1) * 3.0).contiguous()


def _feedforward(torch, ff):
    """feedforward-only commands ff [n, 6] (float32): no position target, zero gains, the model's effort limit"""
    n = ff.shape[0]
    a = torch.zeros((n, 6, 6), device="cuda")
    a[:, :, 0] = float("nan")
    a[:, :, 2] = torch.from_numpy(np.ascontiguousarray(ff, np.float32)).cuda()
    a[:, :, 5] = torch.from_numpy(TAU_MAX).cuda()
    return a


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


def _scale(sim):
    return sim.get_torque_scale_state()[1].cpu().numpy()


def _law(spec, g, k, seed=SEED):
    """[n, 6] the scales of draws k[n] of the envs of global index g"""
    out = np.ones((len(g), 6), dtype=np.float32)
    for kk in np.unique(k):
        sel = k == kk
        out[sel] = scales_np(spec, seed, np.asarray(g)[sel], int(kk))
    return out


# ---- 1. a unit scale changes nothing --------------------------------------------------------------------------------


@pytest.mark.parametrize("extras", [False, True])
@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_unit_scale_changes_nothing(model, torch, kind, mode, extras):
    n, T = 256, 45
    sim = _sim(model, _config(), n, mode, scale=(1.0, 1.0), extras=extras)
    twin = _sim(model, _config(), n, mode, extras=extras)
    same = mode == SAME_STEP
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        for x, y in zip(_step(sim, kind, a, same), _step(twin, kind, a, same)):
            if x is not None:
                assert _bits(x) == _bits(y), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
        if extras and kind == "servos":
            assert _bits(sim.get_history().cpu().numpy()) == _bits(twin.get_history().cpu().numpy()), k
    count, scale = sim.get_torque_scale_state()
    assert count.cpu().numpy().max() > 1  # the episodes did reset
    assert (scale.cpu().numpy() == 1).all()


# ---- 2. the law: a twin fed the scaled torque --------------------------------------------------------------------------


@pytest.mark.parametrize("joints", [ALL, ["left_knee", "right_hip", "right_wheel"]])
def test_twin_fed_the_scaled_torque(model, torch, joints):
    n, T = 512, 60
    cfg = _config()
    sim = _sim(model, cfg, n, SAME_STEP, scale=(0.8, 1.2), joints=joints)
    twin = _sim(model, cfg, n, SAME_STEP)
    rng = np.random.default_rng(11)
    resets = np.zeros(n, dtype=bool)
    contact = 0
    for k in range(T):
        s = _scale(sim)  # the scales this step runs under (a same-step reset draws after the step's physics)
        tau = (rng.uniform(-0.5, 0.5, (n, 6)) * TAU_MAX).astype(np.float32)
        fed = (s * tau).astype(np.float32)  # fl(s * tau)
        x = _step(sim, "servos", _feedforward(torch, tau), same_step=True)
        y = _step(twin, "servos", _feedforward(torch, fed), same_step=True)
        st, tt = _state(sim), _state(twin)
        assert _bits(st[:, OTHER_COLS]) == _bits(tt[:, OTHER_COLS]), k
        assert _bits(st[:, TORQUE_COLS]) == _bits(tau), k
        assert _bits(tt[:, TORQUE_COLS]) == _bits(fed), k
        assert _bits(x[0][:, :, 2]) == _bits(tau) and _bits(y[0][:, :, 2]) == _bits(fed), k  # the torque replies
        assert _bits(x[0][:, :, :2]) == _bits(y[0][:, :, :2]), k
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        done = (x[1] | x[2]).astype(bool)
        assert _bits(x[3][done][:, :, 2]) == _bits(tau[done]), k  # the final observation's replies
        assert _bits(y[3][done][:, :, 2]) == _bits(fed[done]), k
        assert _bits(x[3][done][:, :, :2]) == _bits(y[3][done][:, :, :2]), k
        resets |= done
        contact += int((st[:, _abi.ST_CONTACT] > 0).sum())
    assert resets.mean() > 0.5  # falls and time limits: same-step auto-resets
    assert contact > n * T // 4  # the wheels touched the floor
    mask = sum(1 << ALL.index(j) for j in joints)
    s = _scale(sim)
    assert (s[:, [j for j in range(6) if not (mask >> j) & 1]] == 1).all()
    assert (s[:, [j for j in range(6) if (mask >> j) & 1]] != 1).all()


# ---- 3. draws ----------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_draws_follow_the_law(model, torch, mode):
    n, T, off = 512, 80, 1000
    joints = ["left_hip", "left_knee", "right_wheel"]
    mask = sum(1 << ALL.index(j) for j in joints)
    spec = make_spec(0.7, 1.3, mask)
    sim = _sim(model, _config(max_episode_steps=11), n, mode, scale=(0.7, 1.3), joints=joints, env_offset=off)
    g = off + np.arange(n, dtype=np.uint64)
    expect = np.ones(n, dtype=np.int64)
    pending = np.zeros(n, dtype=bool)
    for k in range(T):
        _, _, term, trunc = sim.step_gyropod(_action(torch, model, "gyropod", n, k))
        done = (term | trunc).cpu().numpy().astype(bool)
        if mode == SAME_STEP:
            expect += done
        else:
            expect += pending
            pending = done
    count, scale = sim.get_torque_scale_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    assert expect.max() > 2
    np.testing.assert_array_equal(scale.cpu().numpy(), _law(spec, g, expect))
    m = torch.zeros(n, dtype=torch.uint8, device="cuda")
    m[::3] = 1
    sim.reset(mask=m, seed=5, env_offset=off)
    expect[m.cpu().numpy().astype(bool)] += 1
    count, scale = sim.get_torque_scale_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(scale.cpu().numpy(), _law(spec, g, expect))
    sim.reset(seed=6, env_offset=off)
    expect += 1
    count, scale = sim.get_torque_scale_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(scale.cpu().numpy(), _law(spec, g, expect))
    init = torch.zeros((n, _abi.INIT_DIM), device="cuda")
    init[:, 2] = 0.6
    init[:, 3] = 1.0
    sim.reset(init_state=init)
    expect += 1
    count, scale = sim.get_torque_scale_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(scale.cpu().numpy(), _law(spec, g, expect))


def test_chunked_host_steps_match_the_device_step(model, torch, monkeypatch):
    from upkie_b200.sim import UpkieSim

    n, T, off = 65536, 25, 77
    cfg = _config(max_episode_steps=6)
    sims = []
    for knobs in ({"HOST_CHUNKS": 5}, {}):
        for k in ("ZERO_COPY", "HOST_CHUNKS", "HOST_SPLIT", "HOST_KERNEL_STREAMS", "HOST_BLOCK", "HOST_BLOCKS_PER_SM"):
            monkeypatch.delenv("UPKIE_B200_" + k, raising=False)
        for k, val in knobs.items():
            monkeypatch.setenv("UPKIE_B200_" + k, str(val))
        s = UpkieSim(n, model=model, config=cfg)
        for k in knobs:
            monkeypatch.delenv("UPKIE_B200_" + k, raising=False)
        s.set_autoreset(SAME_STEP, SEED, off)
        s.set_torque_scale((0.8, 1.2))
        s.reset(seed=SEED, env_offset=off)
        sims.append(s)
    host, dev = sims
    fin_dev = torch.zeros((n, 6, 3), device="cuda")
    resets = np.zeros(n, dtype=bool)
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        obs, term, trunc, fin = (np.array(x, copy=True) for x in host.step_host(
            a.cpu().numpy().reshape(n, 36), 36, compact=True, final_obs=True, final_state=True))
        ro, rt, rr = dev.step_servos_compact_truncated(a, final_obs=fin_dev, final_state=True)
        assert _bits(obs) == _bits(ro.cpu().numpy()), k
        assert _bits(term) == _bits(rt.cpu().numpy()) and _bits(trunc) == _bits(rr.cpu().numpy()), k
        assert _bits(fin) == _bits(fin_dev.cpu().numpy()), k
        assert _bits(host.spine_obs().cpu().numpy()) == _bits(dev.spine_obs().cpu().numpy()), k
        resets |= (term | trunc).astype(bool)
    assert resets[::8192].all() and resets.mean() > 0.5
    for x, y in zip(host.get_torque_scale_state(), dev.get_torque_scale_state()):
        assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy())
    assert _bits(_state(host)) == _bits(_state(dev))
    count, scale = host.get_torque_scale_state()
    count = count.cpu().numpy().astype(np.int64)
    assert count.max() > 2
    spec = make_spec(0.8, 1.2, 0x3F)
    sel = np.arange(0, n, 997)
    np.testing.assert_array_equal(scale.cpu().numpy()[sel], _law(spec, off + sel.astype(np.uint64), count[sel]))


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 30
    whole = _sim(model, _config(), n, SAME_STEP, scale=(0.6, 1.4))
    half = n // 2
    shards = [_sim(model, _config(), half, SAME_STEP, scale=(0.6, 1.4), env_offset=o) for o in (0, half)]
    for k in range(T):
        a = _action(torch, model, "gyropod", n, k)
        out = _step(whole, "gyropod", a)
        for s, o in zip(shards, (0, half)):
            part = _step(s, "gyropod", a[o:o + half].contiguous())
            assert _bits(part[0]) == _bits(out[0][o:o + half]), k
            assert _bits(part[5]) == _bits(out[5][o:o + half]), k
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_torque_scale_state(), whole.get_torque_scale_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o:o + half])


# ---- 4. checkpoints, fixed scales, rejections, None and replacement -----------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 256
    cfg = _config()
    sim = _sim(model, cfg, n, SAME_STEP, scale=(0.7, 1.3), joints=["left_hip", "right_wheel"])
    for k in range(10):
        _step(sim, "servos", _action(torch, model, "servos", n, k), same_step=True)
    sd = sim.state_dict()
    assert sd["torque_scale"][1] == 0b100001
    ref = [_step(sim, "servos", _action(torch, model, "servos", n, 10 + k), same_step=True) for k in range(15)]
    other = UpkieSim(n, model=model, config=cfg)
    other.load_state_dict(sd)
    for k in range(15):
        for x, y in zip(_step(other, "servos", _action(torch, model, "servos", n, 10 + k), same_step=True), ref[k]):
            if x is not None:
                assert _bits(x) == _bits(y), k
    for x, y in zip(other.get_torque_scale_state(), sim.get_torque_scale_state()):
        assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy())
    # a checkpoint written before the feature existed: loads with it off
    for key in ("torque_scale", "torque_scale_count", "torque_scale_scale"):
        del sd[key]
    other.load_state_dict(sd)
    assert other.torque_scale_spec is None


def test_fixed_scales_and_state_rejections(model, torch):
    n = 128
    cfg = _config(max_episode_steps=0, servos_fall_termination=0)
    sim = _sim(model, cfg, n, 0, scale=(1.0, 1.0), joints=["left_knee", "left_wheel"])
    twin = _sim(model, cfg, n, 0)
    s = np.ones((n, 6), dtype=np.float32)
    s[:, 1] = 0.75
    s[:, 2] = np.linspace(0.5, 2.0, n)
    count = torch.full((n,), 4, dtype=torch.int32, device="cuda")
    sim.set_torque_scale_state(count, torch.from_numpy(s).cuda())
    np.testing.assert_array_equal(_scale(sim), s)
    rng = np.random.default_rng(12)
    for k in range(5):
        tau = (rng.uniform(-0.4, 0.4, (n, 6)) * TAU_MAX).astype(np.float32)
        sim.step_servos(_feedforward(torch, tau))
        twin.step_servos(_feedforward(torch, s * tau))
        assert _bits(_state(sim)[:, OTHER_COLS]) == _bits(_state(twin)[:, OTHER_COLS]), k
    for bad in (0.0, -1.0, 2.5, float("nan"), float("inf")):
        b = s.copy()
        b[7, 1] = bad
        with pytest.raises((UpkieException, UpkieRuntimeError), match=r"\(0, 2\]"):
            sim.set_torque_scale_state(count, torch.from_numpy(b).cuda())
    b = s.copy()
    b[3, 4] = 0.9  # right_knee is outside the mask
    with pytest.raises((UpkieException, UpkieRuntimeError), match="outside joint_mask"):
        sim.set_torque_scale_state(count, torch.from_numpy(b).cuda())
    np.testing.assert_array_equal(_scale(sim), s)  # the rejected states were not taken


def test_rejections_none_and_replacement(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import UpkieSim

    n = 64
    sim = _sim(model, _config(), n, NEXT_STEP, scale=(0.7, 1.3), joints=["left_hip", "left_knee"], drop=None)
    for sc, joints, what in (((1.2, 0.8), ALL, "scale_low <= scale_high"),
                             ((0.0, 1.0), ALL, "0 < scale_low"),
                             ((0.5, 2.5), ALL, "scale_high <= 2"),
                             ((float("nan"), 1.0), ALL, "finite"),
                             ((0.8, 1.2), [], "joint_mask")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_torque_scale(sc, joints)
    assert sim.torque_scale_spec[1] == 0b000011  # the previous spec is kept
    for field, value, what in (("joint_limits", 0, "joint_limits"), ("body_contacts", 1, "body_contacts")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_config(_config(**{field: value}))
        other = UpkieSim(n, model=model, config=_config(**{field: value}))
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            other.set_torque_scale((0.8, 1.2))
    spine = UpkieSim(n, model=model, config=_config(spine_mode=1))
    with pytest.raises((UpkieException, UpkieRuntimeError), match="spine_mode"):
        spine.set_torque_scale((0.8, 1.2))
    with pytest.raises(UpkieException, match="torque_scale"):
        B200VectorEnv(8, env_type="gyropod", torque_scale=(1.2, 0.8))
    # a replacement keeps the joints that stay, stores 1 for the joints it drops, and holds the ones it adds at 1
    d = _scale(sim)
    assert (d[:, :2] != 1).all() and (d[:, 2:] == 1).all()
    sim.set_torque_scale([(0.5, 0.6)] * 5 + [(1.5, 1.6)], ["left_hip", "right_wheel"])
    e = _scale(sim)
    np.testing.assert_array_equal(e[:, 0], d[:, 0])
    assert (e[:, 1:] == 1).all()
    sim.reset(seed=SEED)
    e = _scale(sim)
    assert (e[:, 0] >= 0.5).all() and (e[:, 0] <= 0.6).all() and (e[:, 5] >= 1.5).all() and (e[:, 1:5] == 1).all()
    # None: the handle's outputs are a plain twin's
    for k in range(3):
        sim.step_gyropod(_action(torch, model, "gyropod", n, k))
    sim.set_torque_scale(None)
    assert sim.torque_scale_spec is None
    with pytest.raises(UpkieException, match="no torque scales"):
        sim.get_torque_scale_state()
    plain = UpkieSim(n, model=model, config=_config())
    plain.set_autoreset(NEXT_STEP, SEED, 0)
    plain.load_state_dict(sim.state_dict())
    for k in range(20):
        a = _action(torch, model, "gyropod", n, 3 + k)
        x, y = sim.step_gyropod(a), plain.step_gyropod(a)
        for u, w in zip(x, y):
            assert _bits(u.cpu().numpy()) == _bits(w.cpu().numpy()), k


# ---- 5. vector envs ------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200 import make_vec

    n = 64
    env = make_vec("Upkie-B200-" + {"servos": "Servos", "gyropod": "Gyropod", "pendulum": "Pendulum",
                                     "base_velocity": "BaseVelocity"}[env_type], n,
                   torque_scale=(0.85, 1.15), torque_scale_joints=WHEELS)
    env.reset(seed=3)
    count, scale = env.sim.get_torque_scale_state()
    assert (count.cpu().numpy() == 1).all()
    spec = make_spec(0.85, 1.15, 0b100100)
    np.testing.assert_array_equal(scale.cpu().numpy(), _law(spec, np.arange(n, dtype=np.uint64), np.ones(n, np.int64),
                                                            seed=3))
    for _ in range(5):
        env.step(env.action_space.sample())
    env.reset(seed=3)  # a seeded reset repeats its draws
    count2, scale2 = env.sim.get_torque_scale_state()
    assert (count2.cpu().numpy() == 1).all() and _bits(scale2.cpu().numpy()) == _bits(scale.cpu().numpy())
    env.set_torque_scale({"left_hip": (0.9, 1.1), "right_knee": 1.25})
    assert env.sim.torque_scale_spec[1] == 0b010001
    env.reset(seed=4)
    s = _scale(env.sim)
    assert (s[:, 4] == np.float32(1.25)).all() and (s[:, [1, 2, 3, 5]] == 1).all()
    for _ in range(5):
        env.step(env.action_space.sample())
    env.set_torque_scale(None)
    env.step(env.action_space.sample())
