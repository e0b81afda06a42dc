# SPDX-License-Identifier: Apache-2.0
"""Push randomisation on the device (upkie_b200_set_push_randomization): the schedule law after fused and explicit
resets, equivalence with the same forces written from the host (alone and summed with user forces), GPU-count
invariance, checkpoints, the rejections, a cleared spec, and the vector envs."""
import ctypes as C

import numpy as np
import pytest

from upkie_b200 import UpkieRuntimeError, _abi
from test_push_randomization_cpu import NEXT_STEP_RESET, SAME_STEP_RESET, STEP, make_spec, push_schedule_np

pytestmark = pytest.mark.gpu

SEED = 13
SPEC = dict(gap=(0, 6), duration=(1, 5), force=((-30.0, -30.0, -5.0), (30.0, 30.0, 5.0)))


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


def _sim(model, cfg, n, mode, spec=None, env_offset=0, table=False):
    """a handle with the spec set, then reset once: the explicit reset starts every schedule at draw 1"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if table:  # the config's values in a table: the FAM_TABLE kernels
        s.set_env_params(s.get_env_params())
    if spec is not None:
        s.set_push_randomization(spec)
    s.reset(seed=SEED, env_offset=env_offset)
    return s


def _action(torch, model, kind, n, k, env_offset=0, total=None):
    total = total or n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(2000 + k)
    if kind == "servos":
        a = torch.zeros((total, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((total, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((total, 6), device="cuda", generator=gen) * 2 - 1) * 4.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    else:
        a = (torch.rand((total, 1), device="cuda", generator=gen) * 2 - 1) * 2.0
    return a[env_offset : env_offset + n].contiguous()


def _step(sim, kind, a):
    out = sim.step_servos(a) if kind == "servos" else sim.step_pendulum(a)
    return [x.clone() for x in out]


def _code(mode, done):
    """the schedule code of a tick whose env finished (`done`) the previous tick (next step) or this tick (same step)"""
    return np.where(done, NEXT_STEP_RESET if mode == 1 else SAME_STEP_RESET, STEP).astype(np.uint8)


# ---- 1. the law --------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "pendulum"])
@pytest.mark.parametrize("mode", [1, 2])
def test_forces_follow_the_law(model, torch, kind, mode):
    n, T = 2048, 300
    spec = make_spec(**SPEC)
    sim = _sim(model, _config(), n, mode, spec)
    g = np.arange(n)
    ticks = [np.full(n, NEXT_STEP_RESET, dtype=np.uint8)]  # the explicit reset after the spec: a restart from (0, 0)
    reported = []
    done_prev = np.zeros(n, dtype=bool)
    resets = 0
    for k in range(T):
        _, _, term, trunc = _step(sim, kind, _action(torch, model, kind, n, k))
        done = (term | trunc).cpu().numpy().astype(bool)
        ticks.append(_code(mode, done_prev if mode == 1 else done))
        resets += int(ticks[-1][ticks[-1] != STEP].size)
        done_prev = done
        reported.append(sim.get_push_forces().cpu().numpy())
    _, expect, count, timer = push_schedule_np(spec, SEED, g, np.array(ticks))
    np.testing.assert_array_equal(np.array(reported), expect[1:])
    c, t = (x.cpu().numpy().astype(np.uint32) for x in sim.get_push_state())
    np.testing.assert_array_equal(c, count[-1])
    np.testing.assert_array_equal(t, timer[-1])
    assert resets > n  # time limits and falls reset the envs
    pushed = np.any(np.array(reported) != 0, axis=2)
    assert 0.2 < pushed.mean() < 0.8


def test_explicit_masked_reset_restarts(model, torch):
    n = 256
    spec = make_spec(**SPEC)
    sim = _sim(model, _config(max_episode_steps=0, servos_fall_termination=0), n, 0, spec)
    ticks = [np.full(n, NEXT_STEP_RESET, dtype=np.uint8)]
    for k in range(25):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
        ticks.append(np.full(n, STEP, dtype=np.uint8))
    mask = (np.arange(n) % 3 == 0).astype(np.uint8)
    sim.reset(mask=torch.from_numpy(mask).cuda(), seed=SEED)  # device-sampled init rows
    ticks.append(np.where(mask == 1, NEXT_STEP_RESET, STEP).astype(np.uint8))
    _, _, count, timer = push_schedule_np(spec, SEED, np.arange(n), np.array(ticks)[:-1])
    _, _, count2, timer2 = push_schedule_np(spec, SEED, np.arange(n), np.where(mask == 1, NEXT_STEP_RESET, 0)[None],
                                            count[-1], timer[-1])
    c, t = (x.cpu().numpy().astype(np.uint32) for x in sim.get_push_state())
    np.testing.assert_array_equal(np.where(mask == 1, count2[0], count[-1]), c)
    np.testing.assert_array_equal(np.where(mask == 1, 0, timer[-1]), t)
    f = sim.get_push_forces().cpu().numpy()
    assert not f[mask == 1].any()


# ---- 2, 3. the same forces written from the host ---------------------------------------------------------------------


@pytest.mark.parametrize("family", ["table", "body"])
@pytest.mark.parametrize("user", [None, "other", "same"])
@pytest.mark.parametrize("mode", [1, 2])
def test_equal_to_host_written_forces(model, torch, family, user, mode):
    """A twin handle in the same kernel family, whose spec pushes with zero force, fed the schedule's forces (plus the
    user's) through set_external_forces before every tick, steps bit for bit as the push handle"""
    n, T = 1024, 120
    spec = make_spec(**SPEC)
    cfg = _config(body_contacts=1 if family == "body" else 0)
    push = _sim(model, cfg, n, mode, spec)
    # the push handle of the table family runs without a table, its twin with the config's values in one
    twin = _sim(model, cfg, n, mode, make_spec(**dict(SPEC, force=((0.0,) * 3, (0.0,) * 3))), table=(family == "table"))
    user_rows = torch.zeros((n, _abi.NB, 3), device="cuda")
    if user is not None:
        b = 2 if user == "other" else spec.body
        user_rows[:, b] = torch.tensor([7.0, -3.0, 11.0], device="cuda") * torch.linspace(0.5, 1.5, n, device="cuda")[:, None]
        push.set_external_forces(user_rows.clone())
    g = np.arange(n)
    count, timer = np.zeros(n, np.uint32), np.zeros(n, np.uint32)
    _, _, c0, t0 = push_schedule_np(spec, SEED, g, np.full((1, n), NEXT_STEP_RESET), count, timer)
    count, timer = c0[0], t0[0]
    done_prev = np.zeros(n, dtype=bool)
    resets = 0
    for k in range(T):
        code = _code(1, done_prev) if mode == 1 else np.full(n, STEP, np.uint8)
        applied, _, c1, t1 = push_schedule_np(spec, SEED, g, code[None], count, timer)
        rows = user_rows.clone()
        rows[:, spec.body] += torch.from_numpy(applied[0]).cuda()
        twin.set_external_forces(rows)
        a = _action(torch, model, "servos", n, k)
        out_p, out_t = _step(push, "servos", a), _step(twin, "servos", a)
        for x, y in zip(out_p, out_t):
            assert torch.equal(x, y), k
        assert torch.equal(push.get_state(), twin.get_state()), k
        done = (out_p[2] | out_p[3]).cpu().numpy().astype(bool)
        if mode == 2:
            code = _code(2, done)
            _, _, c1, t1 = push_schedule_np(spec, SEED, g, code[None], count, timer)
        count, timer = c1[0], t1[0]
        resets += int(done.sum())
        done_prev = done
    assert resets > 0


# ---- 4. GPU-count invariance ---------------------------------------------------------------------------------------------


def test_shards_reproduce_the_whole_batch(model, torch):
    n, T = 1024, 60
    spec = make_spec(**SPEC)
    whole = _sim(model, _config(), n, 1, spec)
    shards = [_sim(model, _config(), n // 2, 1, spec, env_offset=off) for off in (0, n // 2)]
    for k in range(T):
        _step(whole, "servos", _action(torch, model, "servos", n, k))
        for s, off in zip(shards, (0, n // 2)):
            _step(s, "servos", _action(torch, model, "servos", n // 2, k, off, n))
        f = whole.get_push_forces()
        assert torch.equal(torch.cat([s.get_push_forces() for s in shards]), f), k


# ---- 5. checkpoints ------------------------------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    n = 512
    spec = make_spec(**SPEC)
    a = _sim(model, _config(), n, 2, spec)
    for k in range(30):
        _step(a, "servos", _action(torch, model, "servos", n, k))
    sd = a.state_dict()
    ref = []
    for k in range(30, 60):
        ref.append(_step(a, "servos", _action(torch, model, "servos", n, k)) + [a.get_push_forces()])
    b = _sim(model, _config(), n, 0)
    b.load_state_dict(sd)
    for k in range(30, 60):
        out = _step(b, "servos", _action(torch, model, "servos", n, k)) + [b.get_push_forces()]
        for x, y in zip(out, ref[k - 30]):
            assert torch.equal(x, y), k
    # a checkpoint written before push randomisation existed loads as "off, counters 0"
    old = {k: v for k, v in sd.items() if not k.startswith("push_")}
    b.load_state_dict(old)
    assert b._push_randomization is None
    assert all(not x.any() for x in b.get_push_state())
    _step(b, "servos", _action(torch, model, "servos", n, 0))
    assert not b.get_push_forces().any()


# ---- 6. rejections -------------------------------------------------------------------------------------------------------


def test_rejections_keep_the_previous_spec(model, torch):
    from upkie_b200._lib import lib
    from upkie_b200.sim import UpkieSim

    n = 128
    spec = make_spec(**SPEC)
    sim = _sim(model, _config(max_episode_steps=0, servos_fall_termination=0), n, 0, spec)
    for bad in (dict(body=-1), dict(body=7), dict(gap=(4, 3)), dict(duration=(3, 2)), dict(duration=(0, 2)),
                dict(gap=(0, 2**30 + 1)), dict(force=((0, 0, 0), (float("inf"), 0, 0))),
                dict(force=((float("nan"), 0, 0), (1, 0, 0))), dict(force=((1, 0, 0), (0, 0, 0)))):
        with pytest.raises(UpkieRuntimeError):
            sim.set_push_randomization(make_spec(**dict(SPEC, **bad)))
    # the push body's force of set_external_forces in its body frame, either way round
    with pytest.raises(UpkieRuntimeError):
        sim.set_external_forces(torch.zeros((n, _abi.NB, 3), device="cuda"), 1 << spec.body)
    other = make_spec(**dict(SPEC, body=4))
    sim.set_push_randomization(None)
    sim.set_external_forces(torch.zeros((n, _abi.NB, 3), device="cuda"), 1 << 4)
    with pytest.raises(UpkieRuntimeError):
        sim.set_push_randomization(other)
    sim.set_external_forces(None)
    sim.set_push_randomization(spec)
    # in-kernel rollout transports
    act = _action(torch, model, "servos", n, 0)
    obs = torch.zeros((n, 6, 3), device="cuda")
    term = torch.zeros(n, dtype=torch.uint8, device="cuda")
    obs_ptrs = (C.c_void_p * 1)(obs.data_ptr())
    term_ptrs = (C.c_void_p * 1)(term.data_ptr())
    rc = lib().upkie_b200_step_servos_peers(sim._h, C.c_void_p(act.data_ptr()), obs_ptrs, term_ptrs, 1, sim._stream())
    assert rc == -1  # UPKIE_B200_EINVAL
    # joint_limits = 0, spine mode
    for cfg in (_config(joint_limits=0), _config(spine_mode=1)):
        s = UpkieSim(n, model=model, config=cfg)
        with pytest.raises(UpkieRuntimeError):
            s.set_push_randomization(spec)
        s.close()
    with pytest.raises(UpkieRuntimeError):
        sim.set_config(_config(max_episode_steps=0, servos_fall_termination=0, joint_limits=0))
    # the spec in force is the first one
    ticks = [np.full(n, NEXT_STEP_RESET, dtype=np.uint8)]
    reported = []
    for k in range(40):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
        ticks.append(np.full(n, STEP, dtype=np.uint8))
        reported.append(sim.get_push_forces().cpu().numpy())
    _, expect, _, _ = push_schedule_np(spec, SEED, np.arange(n), np.array(ticks))
    np.testing.assert_array_equal(np.array(reported), expect[1:])


# ---- 7. off ----------------------------------------------------------------------------------------------------------------


def test_cleared_spec_is_off(model, torch):
    n = 512
    a = _sim(model, _config(), n, 1, make_spec(**SPEC), table=True)
    a.set_push_randomization(None)
    b = _sim(model, _config(), n, 1, None, table=True)
    for k in range(60):
        act = _action(torch, model, "servos", n, k)
        for x, y in zip(_step(a, "servos", act), _step(b, "servos", act)):
            assert torch.equal(x, y), k
        assert not a.get_push_forces().any()
    assert torch.equal(a.get_state(), b.get_state())


# ---- 8. vector envs ------------------------------------------------------------------------------------------------------


PUSH_DICT = {"link": "torso", "interval": (0.0, 0.05), "duration": (0.01, 0.03),
             "force": ((-40.0, -40.0, 0.0), (40.0, 40.0, 0.0))}


def test_vector_env_repeats_under_seeded_reset(torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import neutral_action

    n = 256
    env = B200VectorEnv(n, "servos", autoreset_mode="next_step", max_episode_steps=25, push_randomization=PUSH_DICT)
    a = neutral_action(env.model, n, "cuda")

    def run():
        env.reset(seed=5)
        out = []
        for _ in range(60):
            obs, _, term, trunc, _ = env.step_tensors(a)
            out.append((obs.clone(), term.clone(), env.sim.get_push_forces()))
        return out

    first, second = run(), run()
    for x, y in zip(first, second):
        for u, v in zip(x, y):
            assert torch.equal(u, v)
    assert any(f.any() for _, _, f in first)
    env.close()


def test_base_velocity_env_is_pushed(torch):
    from upkie_b200.envs import B200VectorEnv

    n = 64
    envs = [B200VectorEnv(n, "base_velocity", push_randomization=p) for p in (PUSH_DICT, None)]
    states = []
    pushed = False
    for env in envs:
        env.reset(seed=3)
        for _ in range(40):
            env.step(np.zeros((n, 2), dtype=np.float32))
            pushed |= bool(env.sim.get_push_forces().any())
        states.append(env.sim.get_state().cpu().numpy())
    assert pushed
    assert not np.array_equal(states[0], states[1])
    for env in envs:
        env.close()
