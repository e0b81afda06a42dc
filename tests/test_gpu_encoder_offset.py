# SPDX-License-Identifier: Apache-2.0
"""Servo encoder zero offsets on the device (upkie_b200_set_encoder_offset): an UpkieServos handle with offsets is a twin
without them whose position targets are shifted by -delta, reporting positions + delta; zero ranges change nothing;
gyropod and pendulum leg targets start at the reported positions and decay toward the servo zero; same-step terminal
observations keep the terminal episode's offsets; the composition with the observation delay, servo dropouts, the
history and the action delay; the draws follow the NumPy law over fused, explicit, masked, sharded and chunked
host-buffer resets; checkpoints and fixed offsets; the rejections; the vector envs."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_encoder_offset_cpu import offsets_np

pytestmark = pytest.mark.gpu

SEED = 0x0FF5E7
NEXT_STEP, SAME_STEP = 1, 2
ALL = list(_abi.JOINT_NAMES)
LEGS = [0, 1, 3, 4]
LT = slice(_abi.ST_LEG_TARGET, _abi.ST_LEG_TARGET + 4)
POS = [_abi.SP_SERVO + j * 5 for j in range(6)]  # the servo positions of a spine row
# history columns: a hip and a wheel position, the odometry (offset), the pitch (not)
HISTORY = [_abi.SP_SERVO, _abi.SP_SERVO + 2 * 5, _abi.SP_ODOM_POS, _abi.SP_PITCH]
FINAL_SHAPE = {"servos": (6, 5), "gyropod": (6,), "pendulum": (4,)}


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


def _sim(model, cfg, n, mode, offset=None, joints=ALL, history=HISTORY, sense=None, drop=(0.0, 0.0), env_offset=0,
         action_delay=None):
    """a handle reset once; a zero-probability servo-dropout spec runs it in FAM_SENSE, so that a twin without the
    offsets runs the same kernels"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if history:
        s.set_history(history, 5)
    if sense is not None:
        s.set_observation_delay(*sense)
    if drop is not None:
        s.set_servo_dropout(*drop)
    if action_delay is not None:
        s.set_action_delay(*action_delay)
    if offset is not None:
        s.set_encoder_offset(offset[0], offset[1], joints)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(4000 + k)
    if kind == "servos":
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 4.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
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


def _delta(sim):
    return sim.get_encoder_offset_state()[1].cpu().numpy()


def _shifted(a, d):
    """the twin's servo action: the position targets as the offset handle's joints execute them"""
    t = a.clone()
    t[:, :, 0] -= torch_mod.from_numpy(d).cuda()
    return t


def _odometry(model, q2, q5):
    sr = np.float32((1.0 if model.left_wheeled else -1.0) * model.wheel_radius)
    return np.float32(0.5) * (q2 - q5) * sr


def check_spine(model, got, twin, d, label=""):
    """spine rows [n, SPINE_DIM]: the servo positions and the odometry are the twin's read through d, the rest bit for
    bit"""
    np.testing.assert_array_equal(got[:, POS], twin[:, POS] + d, err_msg=label)
    np.testing.assert_allclose(got[:, _abi.SP_ODOM_POS], _odometry(model, twin[:, POS[2]] + d[:, 2],
                                                                  twin[:, POS[5]] + d[:, 5]), atol=1e-6, err_msg=label)
    keep = np.ones(_abi.SPINE_DIM, bool)
    keep[POS + [_abi.SP_ODOM_POS]] = False
    assert _bits(got[:, keep]) == _bits(twin[:, keep]), label


def check_history(model, got, twin, d, label=""):
    for k in range(got.shape[1]):
        np.testing.assert_array_equal(got[:, k, 0], twin[:, k, 0] + d[:, 0], err_msg=label)
        np.testing.assert_array_equal(got[:, k, 1], twin[:, k, 1] + d[:, 2], err_msg=label)
        assert _bits(got[:, k, 3]) == _bits(twin[:, k, 3]), label


# ---- 1. UpkieServos: the shifted twin; 4. episode boundaries -------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_servos_twin(model, torch, mode):
    n, T = 512, 200
    lo, hi = np.asarray(model.q_lower), np.asarray(model.q_upper)
    assert (lo[LEGS] < -0.75).all() and (hi[LEGS] > 0.75).all()  # the targets stay inside the clamps
    cfg = _config()
    sim = _sim(model, cfg, n, mode, offset=(-0.1, 0.1))
    twin = _sim(model, cfg, n, mode)
    same = mode == SAME_STEP
    resets = 0
    for k in range(T):
        d_old = _delta(sim)
        a = _action(torch, model, "servos", n, k)
        x = _step(sim, "servos", a, same)
        y = _step(twin, "servos", _shifted(a, d_old), same)
        d = _delta(sim)
        s, t = _state(sim), _state(twin)
        other = np.ones(_abi.STATE_DIM, bool)
        other[LT] = False
        assert _bits(s[:, other]) == _bits(t[:, other]), k  # get_state's q too
        np.testing.assert_array_equal(s[:, LT], t[:, LT] + d[:, LEGS], err_msg=str(k))  # set by the last reset
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        np.testing.assert_array_equal(x[0][:, :, 0], y[0][:, :, 0] + d, err_msg=str(k))
        assert _bits(x[0][:, :, 1:]) == _bits(y[0][:, :, 1:]), k
        check_spine(model, x[5], y[5], d, str(k))
        check_history(model, x[6], y[6], d, str(k))  # a reset refills with the new offsets
        done = (x[1] | x[2]).astype(bool)
        if same and done.any():
            # the terminal step's observations: the terminal episode's offsets
            np.testing.assert_array_equal(x[3][done][:, :, 0], y[3][done][:, :, 0] + d_old[done], err_msg=str(k))
            check_spine(model, x[4][done], y[4][done], d_old[done], f"final {k}")
            assert (d[done] != d_old[done]).all()
        resets += int(done.sum())
    assert resets > n


# ---- 2. zero ranges -----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_zero_ranges_change_nothing(model, torch, kind, mode):
    n, T = 256, 120
    cfg = _config()
    sim = _sim(model, cfg, n, mode, offset=(0.0, 0.0))
    twin = _sim(model, cfg, n, mode)
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        x = _step(sim, kind, a, mode == SAME_STEP)
        y = _step(twin, kind, a, mode == SAME_STEP)
        for u, v in zip(x, y):
            if u is not None:
                assert _bits(u) == _bits(v), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
    assert (_delta(sim) == 0).all()


# ---- 3. gyropod and pendulum leg targets --------------------------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["gyropod", "pendulum"])
def test_reset_leg_targets_are_the_reported_positions(model, torch, kind, mode):
    n, T = 512, 60
    sim = _sim(model, _config(), n, mode, offset=(-0.1, 0.1), history=None)
    spine = sim.spine_obs().cpu().numpy()
    np.testing.assert_array_equal(_state(sim)[:, LT], spine[:, [POS[j] for j in LEGS]])  # the explicit reset
    resets = 0
    for k in range(T):
        x = _step(sim, kind, _action(torch, model, kind, n, k), mode == SAME_STEP)
        # a same-step reset, and a next-step reset (the step after a termination), start at the reported positions
        done = (x[1] | x[2]).astype(bool) if mode == SAME_STEP else pending if k else np.zeros(n, bool)
        if done.any():
            np.testing.assert_array_equal(_state(sim)[done][:, LT], x[5][done][:, [POS[j] for j in LEGS]])
        resets += int(done.sum())
        pending = (x[1] | x[2]).astype(bool)
    assert resets > 0


@pytest.mark.parametrize("kind", ["gyropod", "pendulum"])
def test_leg_targets_against_a_servos_twin(model, torch, kind):
    """the offset handle's wrapper against an UpkieServos twin without offsets, fed the servo rows gyropod_action
    builds from the offset handle's (decayed) leg targets with the positions shifted by -delta. Zero wheel commands
    keep the wheel rows exact on the host. The two kernels are separate inlined copies of the substep, which fast-math
    may contract differently: within a tolerance."""
    n, T = 256, 200
    cfg = _config(max_episode_steps=0)
    sim = _sim(model, cfg, n, 0, offset=(-0.1, 0.1), history=None)
    twin = _sim(model, cfg, n, 0, history=None)
    twin.set_state(sim.get_state())
    d = torch.from_numpy(_delta(sim)).cuda()
    act = torch.zeros((n, 2 if kind == "gyropod" else 1), device="cuda")
    tau_max = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    phys = np.ones(_abi.STATE_DIM, bool)
    phys[LT] = False
    phys[[_abi.ST_YAW, _abi.ST_YAW_VEL]] = False
    worst = 0.0
    for k in range(T):
        _step(sim, kind, act)
        lt = sim.get_state()[:, LT]
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = float("nan")
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = tau_max
        a[:, LEGS, 0] = lt - d[:, LEGS]
        a[:, LEGS, 3] = a[:, LEGS, 4] = float(cfg.leg_gain_scale)
        twin.step_servos(a)
        s, t = _state(sim)[:, phys], _state(twin)[:, phys]
        worst = max(worst, float(np.nanmax(np.abs(s - t))))
        np.testing.assert_allclose(s, t, atol=1e-5, rtol=1e-5, err_msg=str(k))
    print(f"worst deviation {kind}: {worst:.3g}")


def test_pd_policy_legs_settle_at_the_servo_zero(model, torch):
    """the README's PD policy on UpkiePendulum: after 1 000 ticks the legs of the envs still up stand at the physical
    angle -delta, up to the servos' steady-state error under the robot's weight. Measured on an H100: none of the 1 024
    envs fell, worst |q + delta| 0.0226 rad, and q + delta spreads over the envs about 0.3 times as much as delta (it
    would spread as much if the legs held the joint zero)."""
    from upkie_b200.envs import B200VectorEnv

    n = 1024
    env = B200VectorEnv(n, env_type="pendulum", autoreset_mode="disabled", encoder_offset=(-0.05, 0.05))
    obs, _ = env.reset(seed=3)
    gains = np.array([10.0, 1.0, 0.0, 0.1], dtype=np.float32)
    up = np.ones(n, bool)
    for _ in range(1000):
        obs, _, term, trunc, _ = env.step((np.asarray(obs) @ gains)[:, None].astype(np.float32))
        up &= ~np.asarray(term).astype(bool)
    d = _delta(env.sim)
    q = _state(env.sim)[:, _abi.ST_Q:_abi.ST_Q + 6]
    err = np.abs(q + d)[up][:, LEGS]
    print(f"pendulum PD: {up.sum()} of {n} up, worst |q + delta| {err.max() if up.any() else float('nan'):.3g}")
    assert up.sum() >= n // 4
    assert err.max() < 0.03
    # the legs follow the servo zero, not the joint zero: q + delta varies across envs less than delta does
    qd = (q + d)[up][:, LEGS]
    print(f"std over envs of q + delta {qd.std(axis=0)}, of delta {d[up][:, LEGS].std(axis=0)}")
    assert (qd.std(axis=0) < 0.5 * d[up][:, LEGS].std(axis=0)).all()


# ---- 5. composition ------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("sense", [(0, 0), (2, 2)])
def test_composition(model, torch, sense):
    n, T = 512, 60
    cfg = _config(max_episode_steps=13, nb_substeps=5)
    sims = [_sim(model, cfg, n, SAME_STEP, offset=o, sense=sense, drop=(0.4, 0.4), action_delay=(1, 3))
            for o in ((-0.1, 0.1), None)]
    sim, twin = sims
    resets = 0
    for k in range(T):
        d_old = _delta(sim)
        a = _action(torch, model, "servos", n, k)
        x = _step(sim, "servos", a, True)
        y = _step(twin, "servos", _shifted(a, d_old), True)
        d = _delta(sim)
        other = np.ones(_abi.STATE_DIM, bool)
        other[LT] = False
        assert _bits(_state(sim)[:, other]) == _bits(_state(twin)[:, other]), k
        # the delayed snapshot and the latched servos, read through the offsets
        np.testing.assert_array_equal(x[0][:, :, 0], y[0][:, :, 0] + d, err_msg=str(k))
        assert _bits(x[0][:, :, 1:]) == _bits(y[0][:, :, 1:]), k
        check_spine(model, x[5], y[5], d, str(k))
        check_history(model, x[6], y[6], d, str(k))
        # the action-delay buffers hold the commands as sent: the twin's shifted ones + delta
        cs = sim.get_action_delay_state()[2].cpu().numpy().reshape(n, 6, 6)
        ct = twin.get_action_delay_state()[2].cpu().numpy().reshape(n, 6, 6)
        assert _bits(cs[:, :, 1:]) == _bits(ct[:, :, 1:]), k
        np.testing.assert_allclose(cs[:, :, 0], ct[:, :, 0] + d, atol=1e-6, err_msg=str(k))
        done = (x[1] | x[2]).astype(bool)
        if done.any():
            np.testing.assert_array_equal(x[3][done][:, :, 0], y[3][done][:, :, 0] + d_old[done], err_msg=str(k))
        resets += int(done.sum())
    assert resets > 0
    assert sim.get_servo_dropout_state()[1].cpu().numpy().min() == np.float32(0.4)


# ---- 6. draws on the device -----------------------------------------------------------------------------------------------


def _law(spec, g, k, seed=SEED):
    return np.stack([offsets_np(spec, seed, np.asarray([x], dtype=np.uint64), int(kk))[0] for x, kk in zip(g, k)])


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_draws_follow_the_law(model, torch, mode):
    n, T, off = 512, 80, 1000
    joints = ["left_hip", "left_knee", "right_wheel"]
    spec = _abi.UpkieEncoderOffset(-0.2, 0.1, sum(1 << ALL.index(j) for j in joints), 0)
    sim = _sim(model, _config(max_episode_steps=11), n, mode, offset=(-0.2, 0.1), joints=joints, history=None,
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
    count, offset = sim.get_encoder_offset_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    assert expect.max() > 2
    np.testing.assert_array_equal(offset.cpu().numpy(), _law(spec, g, expect))
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    sim.reset(mask=mask, seed=5, env_offset=off)
    expect[mask.cpu().numpy().astype(bool)] += 1
    count, offset = sim.get_encoder_offset_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(offset.cpu().numpy(), _law(spec, g, expect))
    init = torch.zeros((n, _abi.INIT_DIM), device="cuda")
    init[:, 2] = 0.6
    init[:, 3] = 1.0
    sim.reset(init_state=init)
    expect += 1
    count, offset = sim.get_encoder_offset_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_array_equal(offset.cpu().numpy(), _law(spec, g, expect))


# ---- 7. host paths and shards ---------------------------------------------------------------------------------------------


def test_chunked_host_steps_match_the_device_step(model, torch, monkeypatch):
    from upkie_b200.sim import UpkieSim

    n, T, off = 65536, 25, 77
    cfg = _config(max_episode_steps=6)
    sims = []
    for knobs in ({"HOST_CHUNKS": 5}, {}):
        for k in ("ZERO_COPY", "HOST_CHUNKS", "HOST_SPLIT", "HOST_KERNEL_STREAMS", "HOST_BLOCK", "HOST_BLOCKS_PER_SM"):
            monkeypatch.delenv("UPKIE_B200_" + k, raising=False)
        for k, v in knobs.items():
            monkeypatch.setenv("UPKIE_B200_" + k, str(v))
        s = UpkieSim(n, model=model, config=cfg)
        for k in knobs:
            monkeypatch.delenv("UPKIE_B200_" + k, raising=False)
        s.set_autoreset(SAME_STEP, SEED, off)
        s.set_encoder_offset(-0.1, 0.1, ALL)
        s.reset(seed=SEED, env_offset=off)
        sims.append(s)
    host, dev = sims
    fin_dev = torch.zeros((n, 6, 3), device="cuda")
    resets = np.zeros(n, dtype=bool)
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        obs, term, trunc, fin = (np.array(v, copy=True) for v in host.step_host(
            a.cpu().numpy().reshape(n, 36), 36, compact=True, final_obs=True, final_state=True))
        ro, rt, rr = dev.step_servos_compact_truncated(a, final_obs=fin_dev, final_state=True)
        assert _bits(obs) == _bits(ro.cpu().numpy()), k
        assert _bits(term) == _bits(rt.cpu().numpy()) and _bits(trunc) == _bits(rr.cpu().numpy()), k
        assert _bits(fin) == _bits(fin_dev.cpu().numpy()), k
        assert _bits(host.final_spine_obs().cpu().numpy()) == _bits(dev.final_spine_obs().cpu().numpy()), k
        assert _bits(host.spine_obs().cpu().numpy()) == _bits(dev.spine_obs().cpu().numpy()), k
        resets |= (term | trunc).astype(bool)
    assert resets[::8192].all() and resets.mean() > 0.5
    for u, v in zip(host.get_encoder_offset_state(), dev.get_encoder_offset_state()):
        assert _bits(u.cpu().numpy()) == _bits(v.cpu().numpy())
    count, offset = host.get_encoder_offset_state()
    count = count.cpu().numpy().astype(np.int64)
    assert count.max() > 2
    spec = _abi.UpkieEncoderOffset(-0.1, 0.1, 0x3F, 0)
    sel = np.arange(0, n, 997)
    np.testing.assert_array_equal(offset.cpu().numpy()[sel], _law(spec, off + sel.astype(np.uint64), count[sel]))


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 30
    whole = _sim(model, _config(), n, SAME_STEP, offset=(-0.1, 0.1))
    half = n // 2
    shards = [_sim(model, _config(), half, SAME_STEP, offset=(-0.1, 0.1), env_offset=o) for o in (0, half)]
    for k in range(T):
        a = _action(torch, model, "gyropod", n, k)
        out = _step(whole, "gyropod", a)
        for s, o in zip(shards, (0, half)):
            part = _step(s, "gyropod", a[o:o + half].contiguous())
            assert _bits(part[0]) == _bits(out[0][o:o + half]), k
            assert _bits(part[5]) == _bits(out[5][o:o + half]), k
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_encoder_offset_state(), whole.get_encoder_offset_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o:o + half])


# ---- 8. checkpoints and fixed offsets ---------------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 256
    cfg = _config()
    sim = _sim(model, cfg, n, SAME_STEP, offset=(-0.1, 0.1), joints=["left_hip", "right_knee"])
    for k in range(10):
        _step(sim, "gyropod", _action(torch, model, "gyropod", n, k), same_step=True)
    sd = sim.state_dict()
    assert sd["encoder_offset"] == (np.float32(-0.1), np.float32(0.1), 0b010001)
    ref = [_step(sim, "gyropod", _action(torch, model, "gyropod", n, 10 + k), same_step=True) for k in range(15)]
    other = UpkieSim(n, model=model, config=cfg)
    other.load_state_dict(sd)
    for k in range(15):
        for x, y in zip(_step(other, "gyropod", _action(torch, model, "gyropod", n, 10 + k), same_step=True), ref[k]):
            if x is not None:
                assert _bits(x) == _bits(y), k
    for x, y in zip(other.get_encoder_offset_state(), sim.get_encoder_offset_state()):
        assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy())
    del sd["encoder_offset"]
    other.load_state_dict(sd)
    assert other.encoder_offset_spec is None


def test_fixed_offsets(model, torch):
    n = 128
    cfg = _config(max_episode_steps=0)
    sim = _sim(model, cfg, n, 0, offset=(0.0, 0.0), joints=["left_hip", "left_knee", "left_wheel"], history=None)
    twin = _sim(model, cfg, n, 0, history=None)
    d = np.zeros((n, 6), dtype=np.float32)
    d[:, :3] = np.random.default_rng(2).uniform(-0.3, 0.3, (n, 3))
    count = torch.full((n,), 4, dtype=torch.int32, device="cuda")
    sim.set_encoder_offset_state(count, torch.from_numpy(d).cuda())
    check_spine(model, sim.spine_obs().cpu().numpy(), twin.spine_obs().cpu().numpy(), d)
    ro, rt = sim.reset_obs(_abi.OBS_DIM).cpu().numpy(), twin.reset_obs(_abi.OBS_DIM).cpu().numpy()
    np.testing.assert_array_equal(ro.reshape(n, 6, 5)[:, :, 0], rt.reshape(n, 6, 5)[:, :, 0] + d)
    g6, t6 = sim.reset_obs(6).cpu().numpy(), twin.reset_obs(6).cpu().numpy()
    assert (g6[:, 0] != t6[:, 0]).all() and _bits(g6[:, 1:]) == _bits(t6[:, 1:])
    for bad, what in ((0.6, "0.5"), (float("nan"), "finite")):
        b = d.copy()
        b[7, 1] = bad
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_encoder_offset_state(count, torch.from_numpy(b).cuda())
    b = d.copy()
    b[3, 4] = 0.01  # right_knee is outside the mask
    with pytest.raises((UpkieException, UpkieRuntimeError), match="outside joint_mask"):
        sim.set_encoder_offset_state(count, torch.from_numpy(b).cuda())
    np.testing.assert_array_equal(_delta(sim), d)  # the rejected states were not taken


# ---- 9. rejections, None, mask replacement ------------------------------------------------------------------------------------


def test_rejections_none_and_replacement(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import UpkieSim

    n = 64
    sim = _sim(model, _config(), n, NEXT_STEP, offset=(-0.1, 0.1), history=None, drop=None)
    for lo, hi, joints, what in ((0.1, 0.0, ALL, "low <= high"), (0.0, 0.6, ALL, "0.5"),
                                 (float("nan"), 0.0, ALL, "finite"), (0.0, 0.1, [], "joint_mask")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_encoder_offset(lo, hi, joints)
    assert sim.encoder_offset_spec == (np.float32(-0.1), np.float32(0.1), 0x3F)  # the previous spec is kept
    for field, value, what in (("joint_limits", 0, "joint_limits"), ("body_contacts", 1, "body_contacts")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_config(_config(**{field: value}))
        other = UpkieSim(n, model=model, config=_config(**{field: value}))
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            other.set_encoder_offset(-0.1, 0.1)
    spine = UpkieSim(n, model=model, config=_config(spine_mode=1))
    with pytest.raises((UpkieException, UpkieRuntimeError), match="spine_mode"):
        spine.set_encoder_offset(-0.1, 0.1)
    with pytest.raises(UpkieException, match="encoder_offset"):
        B200VectorEnv(8, env_type="gyropod", encoder_offset=(0.2, 0.1))
    # a replacement zeroes the joints it drops and keeps the others
    d = _delta(sim)
    sim.set_encoder_offset(-0.2, 0.2, ["left_hip", "right_wheel"])
    e = _delta(sim)
    np.testing.assert_array_equal(e[:, [0, 5]], d[:, [0, 5]])
    assert (e[:, [1, 2, 3, 4]] == 0).all()
    # None: the handle's outputs are a plain twin's
    for k in range(3):
        sim.step_gyropod(_action(torch, model, "gyropod", n, k))
    sim.set_encoder_offset(None)
    assert sim.encoder_offset_spec is None
    with pytest.raises(UpkieException, match="no encoder offsets"):
        sim.get_encoder_offset_state()
    plain = UpkieSim(n, model=model, config=_config())
    plain.set_autoreset(NEXT_STEP, SEED, 0)
    plain.load_state_dict(sim.state_dict())
    for k in range(20):
        a = _action(torch, model, "gyropod", n, 3 + k)
        x, y = sim.step_gyropod(a), plain.step_gyropod(a)
        for u, v in zip(x, y):
            assert _bits(u.cpu().numpy()) == _bits(v.cpu().numpy()), k
        assert _bits(sim.spine_obs().cpu().numpy()) == _bits(plain.spine_obs().cpu().numpy()), k


# ---- 10. vector envs ----------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200 import make_vec

    n = 64
    env = make_vec("Upkie-B200-" + {"servos": "Servos", "gyropod": "Gyropod", "pendulum": "Pendulum",
                                     "base_velocity": "BaseVelocity"}[env_type], n, encoder_offset=0.05)
    env.reset(seed=3)
    count, offset = env.sim.get_encoder_offset_state()
    assert (count.cpu().numpy() == 1).all()
    spec = _abi.UpkieEncoderOffset(-0.05, 0.05, 0b011011, 0)
    np.testing.assert_array_equal(offset.cpu().numpy(), _law(spec, np.arange(n, dtype=np.uint64), np.ones(n, np.int64),
                                                             seed=3))
    d = offset.cpu().numpy()
    q = _state(env.sim)[:, _abi.ST_Q:_abi.ST_Q + 6]
    spine = env.sim.spine_obs().cpu().numpy()
    np.testing.assert_array_equal(spine[:, POS], q + d)
    np.testing.assert_array_equal(_state(env.sim)[:, LT], (q + d)[:, LEGS])
    for _ in range(5):
        env.step(env.action_space.sample())
    env.set_encoder_offset(None)
    env.step(env.action_space.sample())
