# SPDX-License-Identifier: Apache-2.0
"""Servo velocity limits on the device (upkie_b200_set_velocity_derate): the reported torque is the NumPy law applied to
the set joint velocities; limits no joint reaches change nothing, alone and with the action delay, servo noise and
encoder offsets; a free wheel saturates within its drawn limit and band while its twin does not; the draws follow the
NumPy law over fused, explicit, masked, sharded and chunked host-buffer resets; checkpoints and fixed limits; the
rejections, None and replacement; the vector envs."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_velocity_derate_cpu import TAU_MAX, law_np, limits_np, make_spec

pytestmark = pytest.mark.gpu

SEED = 0x7E10C
NEXT_STEP, SAME_STEP = 1, 2
ALL = list(_abi.JOINT_NAMES)
WHEELS = ["left_wheel", "right_wheel"]
FINAL_SHAPE = {"servos": (6, 5), "gyropod": (6,), "pendulum": (4,)}
HISTORY = [_abi.SP_SERVO + 1, _abi.SP_SERVO + 2, _abi.SP_ODOM_VEL, _abi.SP_PITCH]  # a velocity and a torque reply
LOOSE = ((150.0, 200.0), 10.0)  # limits above max_coordinate_velocity: no joint reaches them


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


def _sim(model, cfg, n, mode, vlim=None, joints=ALL, drop=(0.0, 0.0), env_offset=0, extras=False):
    """a handle reset once; a zero-probability servo-dropout spec runs it in FAM_SENSE, so that a twin without the
    limits runs the same kernels. `extras`: the action delay, servo noise and encoder offsets on too"""
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
    if vlim is not None:
        s.set_velocity_derate(vlim[0], vlim[1], joints)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(9000 + k)
    if kind == "servos":
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 20.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
        return a
    dim = 2 if kind == "gyropod" else 1
    return ((torch.rand((n, dim), device="cuda", generator=gen) * 2 - 1) * 3.0).contiguous()


def _feedforward(torch, n, sign):
    """every joint under pure feedforward sign * tau_max (sign: [n, 6] or a number)"""
    a = torch.zeros((n, 6, 6), device="cuda")
    a[:, :, 0] = float("nan")
    a[:, :, 2] = torch.as_tensor(np.asarray(sign * TAU_MAX, np.float32), device="cuda")
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


def _vmax(sim):
    return sim.get_velocity_derate_state()[1].cpu().numpy()


def _law(spec, g, k, seed=SEED):
    """[n, 6] the limits of draws k[n] of the envs of global index g"""
    out = np.zeros((len(g), 6), dtype=np.float32)
    for kk in np.unique(k):
        sel = k == kk
        out[sel] = limits_np(spec, seed, np.asarray(g)[sel], int(kk))
    return out


# ---- 1. the law on the device ---------------------------------------------------------------------------------------


def test_law_on_the_device(model, torch):
    n = 512
    cfg = _config(nb_substeps=1, max_episode_steps=0)
    sim = _sim(model, cfg, n, 0, vlim=((10.0, 10.0), 8.0))
    v = np.array([10.0, 11.0, 40.0, 12.0, 13.0, 45.0], np.float32)
    band = np.array([8.0, 5.0, 20.0, 6.0, 9.0, 12.0], np.float32)
    spec = make_spec(v, v, band, 0x3F)
    sim.set_velocity_derate([(x, x) for x in v], band, ALL)
    sim.set_velocity_derate_state(torch.ones(n, dtype=torch.int32, device="cuda"),
                                  torch.from_numpy(np.tile(v, (n, 1))).cuda())
    assert spec.joint_mask == sim.velocity_derate_spec[2]
    rng = np.random.default_rng(3)
    # joint velocities below, inside and past each joint's band, of both signs, and +-0
    frac = rng.uniform(0.0, 2.5, (n, 6)).astype(np.float32)
    qd = (frac * (v + band) * rng.choice([-1.0, 1.0], (n, 6))).astype(np.float32)
    qd[:8] = 0.0
    qd[8:16] = -0.0
    sign = rng.choice([-1.0, 1.0], (n, 6)).astype(np.float32)
    st = _state(sim)
    st[:, _abi.ST_QD:_abi.ST_QD + 6] = qd
    sim.set_state(torch.from_numpy(st).cuda())
    obs = sim.step_servos(_feedforward(torch, n, sign))[0].cpu().numpy()
    t = sign * TAU_MAX
    ref = law_np(t, qd, v, band, TAU_MAX)
    got = obs[:, :, 2]
    exact = (np.abs(qd) <= v) | (t * qd < 0)
    assert _bits(got[exact]) == _bits(ref[exact])  # below the limit and braking: the command, bit for bit
    # fast-math division: a few ulps of the effort limit
    np.testing.assert_allclose(got, ref, rtol=0, atol=float(4 * np.spacing(np.float32(16.0))))
    derated = ~exact & (np.abs(qd) < v + band)
    assert derated.sum() > 100 and (np.abs(got[derated]) < TAU_MAX[np.where(derated)[1]]).all()
    assert (got[~exact & (np.abs(qd) >= v + band)] == 0).all()


# ---- 2. nothing changes when nothing binds ------------------------------------------------------------------------


@pytest.mark.parametrize("extras", [False, True])
@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_loose_limits_change_nothing(model, torch, kind, mode, extras):
    n, T = 256, 45
    sim = _sim(model, _config(), n, mode, vlim=LOOSE, extras=extras)
    twin = _sim(model, _config(), n, mode, extras=extras)
    same = mode == SAME_STEP
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        for x, y in zip(_step(sim, kind, a, same), _step(twin, kind, a, same)):
            if x is not None:
                assert _bits(x) == _bits(y), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
    assert sim.get_velocity_derate_state()[0].cpu().numpy().max() > 1  # the episodes did reset


# ---- 3. saturation of a free wheel -----------------------------------------------------------------------------------


def test_free_wheels_saturate_within_their_drawn_band(model, torch):
    n = 1024
    cfg = _config(gravity=0.0, max_episode_steps=0, servos_fall_termination=0)
    derate = 10.0
    sim = _sim(model, cfg, n, 0, vlim=((15.0, 40.0), derate), joints=WHEELS)
    twin = _sim(model, cfg, n, 0)
    init = torch.zeros((n, _abi.INIT_DIM), device="cuda")
    init[:, 2] = 1.2  # clear of the floor
    init[:, 3] = 1.0
    sim.reset(init_state=init)
    twin.reset(init_state=init)
    a = _feedforward(torch, n, np.array([0, 0, 1, 0, 0, 1], np.float32))
    a[:, [0, 1, 3, 4], 2] = 0.0  # the legs stay unpowered
    v = _vmax(sim)
    assert (v[:, [0, 1, 3, 4]] == 0).all() and (v[:, 2] >= 15).all() and (v[:, 2] <= 40).all()
    h = 1.0 / (200.0 * cfg.nb_substeps)
    step_gain = TAU_MAX[2] * h / float(np.asarray(model.inertia)[3][1])
    peak = np.zeros((n, 2), np.float32)
    tpeak = np.zeros((n, 2), np.float32)
    for _ in range(40):
        sim.step_servos(a)
        twin.step_servos(a)
        peak = np.maximum(peak, np.abs(_state(sim)[:, [_abi.ST_QD + 2, _abi.ST_QD + 5]]))
        tpeak = np.maximum(tpeak, np.abs(_state(twin)[:, [_abi.ST_QD + 2, _abi.ST_QD + 5]]))
    bound = v[:, [2, 5]] + derate + step_gain
    assert (peak <= bound).all()
    assert (peak > v[:, [2, 5]]).all()  # each wheel does pass its own limit
    assert (tpeak > bound).all()


# ---- 4. draws ----------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_draws_follow_the_law(model, torch, mode):
    n, T, off = 512, 80, 1000
    joints = ["left_hip", "left_knee", "right_wheel"]
    mask = sum(1 << ALL.index(j) for j in joints)
    spec = make_spec(10.0, 30.0, 6.0, mask)
    sim = _sim(model, _config(max_episode_steps=11), n, mode, vlim=((10.0, 30.0), 6.0), joints=joints,
               env_offset=off)
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
    count, vmax = sim.get_velocity_derate_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    assert expect.max() > 2
    np.testing.assert_array_equal(vmax.cpu().numpy(), _law(spec, g, expect))
    m = torch.zeros(n, dtype=torch.uint8, device="cuda")
    m[::3] = 1
    sim.reset(mask=m, seed=5, env_offset=off)
    expect[m.cpu().numpy().astype(bool)] += 1
    count, vmax = sim.get_velocity_derate_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(vmax.cpu().numpy(), _law(spec, g, expect))
    init = torch.zeros((n, _abi.INIT_DIM), device="cuda")
    init[:, 2] = 0.6
    init[:, 3] = 1.0
    sim.reset(init_state=init)
    expect += 1
    count, vmax = sim.get_velocity_derate_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(vmax.cpu().numpy(), _law(spec, g, expect))


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
        s.set_velocity_derate((4.0, 12.0), 3.0, ALL)  # limits the random velocity targets pass
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
    for x, y in zip(host.get_velocity_derate_state(), dev.get_velocity_derate_state()):
        assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy())
    count, vmax = host.get_velocity_derate_state()
    count = count.cpu().numpy().astype(np.int64)
    assert count.max() > 2
    spec = make_spec(4.0, 12.0, 3.0, 0x3F)
    sel = np.arange(0, n, 997)
    np.testing.assert_array_equal(vmax.cpu().numpy()[sel], _law(spec, off + sel.astype(np.uint64), count[sel]))


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 30
    vlim = ((5.0, 15.0), 4.0)
    whole = _sim(model, _config(), n, SAME_STEP, vlim=vlim)
    half = n // 2
    shards = [_sim(model, _config(), half, SAME_STEP, vlim=vlim, env_offset=o) for o in (0, half)]
    for k in range(T):
        a = _action(torch, model, "gyropod", n, k)
        out = _step(whole, "gyropod", a)
        for s, o in zip(shards, (0, half)):
            part = _step(s, "gyropod", a[o:o + half].contiguous())
            assert _bits(part[0]) == _bits(out[0][o:o + half]), k
            assert _bits(part[5]) == _bits(out[5][o:o + half]), k
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_velocity_derate_state(), whole.get_velocity_derate_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o:o + half])


# ---- 5. checkpoints, fixed limits, rejections, None and replacement ---------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 256
    cfg = _config()
    sim = _sim(model, cfg, n, SAME_STEP, vlim=((4.0, 9.0), 2.0), joints=["left_hip", "right_wheel"])
    for k in range(10):
        _step(sim, "servos", _action(torch, model, "servos", n, k), same_step=True)
    sd = sim.state_dict()
    assert sd["velocity_derate"][2] == 0b100001
    ref = [_step(sim, "servos", _action(torch, model, "servos", n, 10 + k), same_step=True) for k in range(15)]
    other = UpkieSim(n, model=model, config=cfg)
    other.load_state_dict(sd)
    for k in range(15):
        for x, y in zip(_step(other, "servos", _action(torch, model, "servos", n, 10 + k), same_step=True), ref[k]):
            if x is not None:
                assert _bits(x) == _bits(y), k
    for x, y in zip(other.get_velocity_derate_state(), sim.get_velocity_derate_state()):
        assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy())
    del sd["velocity_derate"]
    other.load_state_dict(sd)
    assert other.velocity_derate_spec is None


def test_fixed_limits_and_state_rejections(model, torch):
    n = 128
    cfg = _config(max_episode_steps=0, nb_substeps=1)
    sim = _sim(model, cfg, n, 0, vlim=((20.0, 20.0), 5.0), joints=["left_knee", "left_wheel"])
    v = np.zeros((n, 6), dtype=np.float32)
    v[:, 1] = 3.0
    v[:, 2] = np.linspace(2.0, 30.0, n)
    count = torch.full((n,), 4, dtype=torch.int32, device="cuda")
    sim.set_velocity_derate_state(count, torch.from_numpy(v).cuda())
    st = _state(sim)
    st[:, _abi.ST_QD + 2] = 10.0
    sim.set_state(torch.from_numpy(st).cuda())
    obs = sim.step_servos(_feedforward(torch, n, 1.0))[0].cpu().numpy()
    ref = law_np(TAU_MAX[2], np.float32(10.0), v[:, 2], np.float32(5.0), TAU_MAX[2])
    np.testing.assert_allclose(obs[:, 2, 2], ref, rtol=0, atol=float(4 * np.spacing(np.float32(TAU_MAX[2]))))
    for bad, what in ((0.0, "> 0"), (-1.0, "> 0"), (float("nan"), "finite"), (float("inf"), "finite")):
        b = v.copy()
        b[7, 1] = bad
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_velocity_derate_state(count, torch.from_numpy(b).cuda())
    b = v.copy()
    b[3, 4] = 10.0  # right_knee is outside the mask
    with pytest.raises((UpkieException, UpkieRuntimeError), match="outside joint_mask"):
        sim.set_velocity_derate_state(count, torch.from_numpy(b).cuda())
    np.testing.assert_array_equal(_vmax(sim), v)  # the rejected states were not taken


def test_rejections_none_and_replacement(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import UpkieSim

    n = 64
    sim = _sim(model, _config(), n, NEXT_STEP, vlim=((10.0, 20.0), 5.0), joints=["left_hip", "left_knee"], drop=None)
    for mv, d, joints, what in (((20.0, 10.0), 5.0, ALL, "max_velocity_low <= max_velocity_high"),
                                ((0.0, 10.0), 5.0, ALL, "0 < max_velocity_low"),
                                ((10.0, 20.0), 0.0, ALL, "derate > 0"),
                                ((float("nan"), 10.0), 5.0, ALL, "finite"),
                                ((10.0, 20.0), 5.0, [], "joint_mask")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_velocity_derate(mv, d, joints)
    assert sim.velocity_derate_spec[2] == 0b000011  # the previous spec is kept
    for field, value, what in (("joint_limits", 0, "joint_limits"), ("body_contacts", 1, "body_contacts")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_config(_config(**{field: value}))
        other = UpkieSim(n, model=model, config=_config(**{field: value}))
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            other.set_velocity_derate((10.0, 20.0), 5.0)
    spine = UpkieSim(n, model=model, config=_config(spine_mode=1))
    with pytest.raises((UpkieException, UpkieRuntimeError), match="spine_mode"):
        spine.set_velocity_derate((10.0, 20.0), 5.0)
    with pytest.raises(UpkieException, match="velocity_derate"):
        B200VectorEnv(8, env_type="gyropod", velocity_derate={"max_velocity": (20.0, 10.0)})
    # a replacement zeroes the joints it drops, keeps the others, and holds the joints it adds at their high bound
    d = _vmax(sim)
    assert (d[:, :2] >= 10).all() and (d[:, 2:] == 0).all()
    sim.set_velocity_derate([(1.0, 2.0), (1.0, 2.0), (1.0, 2.0), (1.0, 2.0), (1.0, 2.0), (30.0, 50.0)], 5.0,
                            ["left_hip", "right_wheel"])
    e = _vmax(sim)
    np.testing.assert_array_equal(e[:, 0], d[:, 0])
    assert (e[:, [1, 2, 3, 4]] == 0).all() and (e[:, 5] == 50.0).all()
    # None: the handle's outputs are a plain twin's
    for k in range(3):
        sim.step_gyropod(_action(torch, model, "gyropod", n, k))
    sim.set_velocity_derate(None)
    assert sim.velocity_derate_spec is None
    with pytest.raises(UpkieException, match="no velocity limits"):
        sim.get_velocity_derate_state()
    plain = UpkieSim(n, model=model, config=_config())
    plain.set_autoreset(NEXT_STEP, SEED, 0)
    plain.load_state_dict(sim.state_dict())
    for k in range(20):
        a = _action(torch, model, "gyropod", n, 3 + k)
        x, y = sim.step_gyropod(a), plain.step_gyropod(a)
        for u, w in zip(x, y):
            assert _bits(u.cpu().numpy()) == _bits(w.cpu().numpy()), k


# ---- 6. vector envs ------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200 import make_vec
    from upkie_b200.envs import UPKIE_VELOCITY_DERATE, velocity_derate_spec

    n = 64
    env = make_vec("Upkie-B200-" + {"servos": "Servos", "gyropod": "Gyropod", "pendulum": "Pendulum",
                                     "base_velocity": "BaseVelocity"}[env_type], n,
                   velocity_derate={"max_velocity": (10.0, 14.0), "derate": 6.0},
                   velocity_derate_joints=["left_hip", "left_knee", "right_hip", "right_knee"])
    env.reset(seed=3)
    count, vmax = env.sim.get_velocity_derate_state()
    assert (count.cpu().numpy() == 1).all()
    spec = make_spec(10.0, 14.0, 6.0, 0b011011)
    np.testing.assert_array_equal(vmax.cpu().numpy(), _law(spec, np.arange(n, dtype=np.uint64), np.ones(n, np.int64),
                                                           seed=3))
    for _ in range(5):
        env.step(env.action_space.sample())
    env.reset(seed=3)  # a seeded reset repeats its draws
    count2, vmax2 = env.sim.get_velocity_derate_state()
    assert (count2.cpu().numpy() == 1).all() and _bits(vmax2.cpu().numpy()) == _bits(vmax.cpu().numpy())
    env.set_velocity_derate(UPKIE_VELOCITY_DERATE)
    assert env.sim.velocity_derate_spec[2] == 0x3F
    env.reset(seed=4)
    np.testing.assert_array_equal(_vmax(env.sim), np.tile(np.asarray(
        velocity_derate_spec(UPKIE_VELOCITY_DERATE).max_velocity_low, np.float32), (n, 1)))
    for _ in range(5):
        env.step(env.action_space.sample())
    env.set_velocity_derate(None)
    env.step(env.action_space.sample())
