# SPDX-License-Identifier: Apache-2.0
"""Action-delay randomisation on the device (upkie_b200_set_action_delay): a zero delay changes nothing, a full tick
of delay is a one-tick shift of the commands, repeated commands are unaffected, the draws after fused and explicit
resets follow the law on whole and sharded batches, partial delays match the CPU build of the kernels' substeps,
checkpoints, the rejections, a cleared spec, and the vector envs."""
import ctypes as C

import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from conftest import random_servo_actions, random_states
from test_action_delay_cpu import _lib as _cpu_lib, _p, action_delay_draw_np

pytestmark = pytest.mark.gpu

SEED = 29


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


def _sim(model, cfg, n, mode, delay=None, env_offset=0, table=False):
    """a handle with the delay range set, then reset once: the explicit reset draws every env's first delay"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if table:  # the config's values in a table: the FAM_TABLE kernels
        s.set_env_params(s.get_env_params())
    if delay is not None:
        s.set_action_delay(*delay)
    s.reset(seed=SEED, env_offset=env_offset)
    # the host-buffer steps run on the handle's own streams: the set-up enqueued on the caller's stream ends first
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k, env_offset=0, total=None):
    total = total or n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(4000 + k)
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


def _step(sim, kind, a, path="device"):
    if path == "host":
        a = a.cpu().numpy()
        out = sim.step_servos_host(a) if kind == "servos" else sim.step_gyropod_host(a)
        return [np.array(x, copy=True) for x in out]
    out = {"servos": sim.step_servos, "gyropod": sim.step_gyropod, "pendulum": sim.step_pendulum}[kind](a)
    return [x.clone().cpu().numpy() for x in out]


def _bits(x):
    return np.ascontiguousarray(x).tobytes()


# ---- 1. a zero delay changes nothing -----------------------------------------------------------------------------------


@pytest.mark.parametrize("body", [False, True])
@pytest.mark.parametrize("path", ["device", "host"])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_zero_delay_changes_nothing(model, torch, kind, mode, path, body):
    n, T = 512, 70
    cfg = _config(body_contacts=1 if body else 0)
    delayed = _sim(model, cfg, n, mode, (0, 0))
    twin = _sim(model, cfg, n, mode, table=not body)  # FAM_TABLE (FAM_BODY with body contacts)
    # The host-buffer (TILE=1) kernels of FAM_DELAY and FAM_TABLE are separately compiled copies of the same physics.
    # For some (env type, auto-reset) pairs their fp32 results differ in the last bits, which the contact solve can
    # grow within a tick (up to 1.3e-5 on a joint velocity from the same state, measured on an H100). The device-buffer
    # and body-contact copies match bit for bit. On the host path without body contacts the twin is put back on the
    # delayed handle's state before every tick, so that each tick, resets included, is compared from the same state:
    # integer outputs bit for bit, observations within fp32 round-off of one tick (test_gpu_sim_parity.py allows 2e-4
    # on joint angles and 2e-2 on joint rates against the fp64 oracle).
    resync = path == "host" and not body
    resets = 0
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        if resync:
            twin.set_state(delayed.get_state())
            torch.cuda.synchronize()
        out_d = _step(delayed, kind, a, path)
        out_t = _step(twin, kind, a, path)
        for x, y in zip(out_d, out_t):
            if resync and x.dtype == np.float32:
                np.testing.assert_allclose(x, y, rtol=1e-5, atol=1e-3, err_msg=str(k))
            else:
                assert _bits(x) == _bits(y), k
        resets += int(((out_d[2] != 0) | (out_d[3] != 0)).sum())
    if not resync:
        assert _bits(delayed.get_state().cpu().numpy()) == _bits(twin.get_state().cpu().numpy())
    assert resets > 0  # falls or time limits happened
    count, delay, _ = delayed.get_action_delay_state()
    assert not delay.any()
    if mode:
        assert int(count.sum()) > n  # fused resets drew


# ---- 2. a full tick of delay is a one-tick shift -----------------------------------------------------------------------


def test_full_tick_is_a_one_tick_shift(model, torch):
    from upkie_b200.sim import stop_commands

    n, T, nb = 512, 40, 5
    cfg = _config(max_episode_steps=0, servos_fall_termination=0, nb_substeps=nb)
    delayed = _sim(model, cfg, n, 0, (nb, nb))
    twin = _sim(model, cfg, n, 0, (0, 0))
    prev = stop_commands(n, "cuda")
    for k in range(T):
        a = _action(torch, model, "servos", n, k)
        out_d = _step(delayed, "servos", a)
        out_t = _step(twin, "servos", prev)
        for x, y in zip(out_d, out_t):
            assert _bits(x) == _bits(y), k
        prev = a
    assert _bits(delayed.get_state().cpu().numpy()) == _bits(twin.get_state().cpu().numpy())


# ---- 3. identical consecutive commands are unaffected ------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "gyropod"])
def test_repeated_command_is_unaffected(model, torch, kind):
    n, T, nb = 512, 30, 5
    cfg = _config(max_episode_steps=0, servos_fall_termination=0, fall_pitch=10.0)
    delayed = _sim(model, cfg, n, 0, (0, nb))
    twin = _sim(model, cfg, n, 0, (0, 0))
    a = _action(torch, model, kind if kind == "servos" else "pendulum", n, 0)
    if kind == "gyropod":
        a = torch.zeros((n, 2), device="cuda")  # zero velocities: the leg filter at rest gives the same row each tick
    # the command the first tick computes, made the previous command of the delayed handle
    probe = _sim(model, cfg, n, 0, (0, 0))
    _step(probe, kind, a)
    count, delay, _ = delayed.get_action_delay_state()
    _, _, command = probe.get_action_delay_state()
    delayed.set_action_delay_state(count, delay, command)
    assert delay.min() == 0 and delay.max() == nb
    for k in range(T):
        out_d = _step(delayed, kind, a)
        out_t = _step(twin, kind, a)
        for x, y in zip(out_d, out_t):
            assert _bits(x) == _bits(y), k


# ---- 4. the draws ---------------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "pendulum"])
@pytest.mark.parametrize("mode", [1, 2])
def test_draws_follow_the_law(model, torch, kind, mode):
    n, T, low, high = 1024, 150, 0, 5
    sim = _sim(model, _config(), n, mode, (low, high))
    g = np.arange(n, dtype=np.uint64)
    expect = np.ones(n, dtype=np.uint64)  # the explicit reset after the spec: draw 1
    done_prev = np.zeros(n, dtype=bool)
    for k in range(T):
        _, _, term, trunc = _step(sim, kind, _action(torch, model, kind, n, k))
        done = (term | trunc).astype(bool)
        expect += (done_prev if mode == 1 else done).astype(np.uint64)
        done_prev = done
    count, delay, command = (x.cpu().numpy() for x in sim.get_action_delay_state())
    np.testing.assert_array_equal(count.astype(np.uint64), expect)
    np.testing.assert_array_equal(delay.astype(np.uint32), action_delay_draw_np(low, high, SEED, g, expect))
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
        count, delay, command = (x.cpu().numpy() for x in sim.get_action_delay_state())
        np.testing.assert_array_equal(count.astype(np.uint64), expect)
        np.testing.assert_array_equal(delay.astype(np.uint32), action_delay_draw_np(low, high, SEED, g, expect))
        stopped = command[mask == 1]
        assert np.all(np.isnan(stopped[:, :, 0])) and not stopped[:, :, 1:].any()


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 80
    whole = _sim(model, _config(), n, 2, (0, 5))
    half = n // 2
    shards = [_sim(model, _config(), half, 2, (0, 5), env_offset=o) for o in (0, half)]
    for k in range(T):
        out = _step(whole, "servos", _action(torch, model, "servos", n, k))
        for s, o in zip(shards, (0, half)):
            part = _step(s, "servos", _action(torch, model, "servos", half, k, env_offset=o, total=n))
            assert _bits(part[0]) == _bits(out[0][o : o + half])
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_action_delay_state(), whole.get_action_delay_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o : o + half])


# ---- 5. partial delays against the CPU build -----------------------------------------------------------------------------


def test_partial_delays_match_the_cpu_build(model, torch):
    """The fp64 oracle steps whole ticks only: the delayed tick is checked against the kernels' arithmetic compiled for
    the CPU (tests/hostsim/action_delay.cpp), the substeps before the switch under the previous command and the rest
    under the tick's own, within the one-tick tolerances of test_gpu_sim_parity.py."""
    from upkie_b200.sim import UpkieSim

    n, nb = 2048, 5
    cfg = _abi.default_sim_config()
    st32 = random_states(n, seed=3).astype(np.float32)
    act32 = random_servo_actions(n, model, seed=4).astype(np.float32).reshape(n, 36)
    prev32 = random_servo_actions(n, model, seed=5).astype(np.float32).reshape(n, 36)
    L = _cpu_lib()
    m = model.to_struct()
    h = L.hostsim_create(C.byref(m), C.byref(cfg))
    try:
        for d in range(1, nb):
            sim = UpkieSim(n, model=model, config=cfg)
            sim.set_action_delay(d, d)
            sim.set_state(torch.from_numpy(st32).cuda())
            count = torch.zeros(n, dtype=torch.int32, device="cuda")
            delay = torch.full((n,), d, dtype=torch.int32, device="cuda")
            sim.set_action_delay_state(count, delay, torch.from_numpy(prev32.reshape(n, 6, 6)).cuda())
            sim.step_servos(torch.from_numpy(act32.reshape(n, 6, 6)).cuda())
            gs = sim.get_state().cpu().numpy().astype(np.float64)
            cs = st32.copy()
            prev = prev32.copy()
            dl = np.full(n, d, dtype=np.uint32)
            L.hostsim_action_delay_tick(h, n, 0, _p(cs), _p(prev), _p(act32.copy()), dl.ctypes.data_as(
                C.POINTER(C.c_uint32)), 0, 1, 0, None)
            cs = cs.astype(np.float64)
            assert np.abs(gs[:, :7] - cs[:, :7]).max() < 2e-5
            assert np.abs(gs[:, 13:19] - cs[:, 13:19]).max() < 2e-4
            assert np.abs(gs[:, 7:13] - cs[:, 7:13]).max() < 1e-3
            assert np.abs(gs[:, 19:25] - cs[:, 19:25]).max() < 2e-2
            assert np.median(np.abs(gs[:, 19:25] - cs[:, 19:25]).max(axis=1)) < 5e-4
            # the delay is seen: the undelayed tick lands elsewhere
            und = st32.copy()
            prev = prev32.copy()
            L.hostsim_action_delay_tick(h, n, 0, _p(und), _p(prev), _p(act32.copy()), np.zeros(n, np.uint32).ctypes
                                        .data_as(C.POINTER(C.c_uint32)), 0, 1, 0, None)
            assert np.abs(und[:, 19:25] - cs[:, 19:25]).max() > 1e-2
            sim.close()
    finally:
        L.hostsim_destroy(h)


# ---- 6. checkpoints and the API ----------------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n, T = 512, 30
    a = _sim(model, _config(), n, 1, (1, 4))
    for k in range(T):
        _step(a, "servos", _action(torch, model, "servos", n, k))
    sd = a.state_dict()
    assert sd["action_delay"] == (1, 4)
    b = UpkieSim(n, model=model, config=_config())
    b.load_state_dict(sd)
    for k in range(T, 2 * T):
        x = _step(a, "servos", _action(torch, model, "servos", n, k))
        y = _step(b, "servos", _action(torch, model, "servos", n, k))
        for u, v in zip(x, y):
            assert _bits(u) == _bits(v), k
    for u, v in zip(a.get_action_delay_state(), b.get_action_delay_state()):
        assert _bits(u.cpu().numpy()) == _bits(v.cpu().numpy())
    # a checkpoint written before the feature: off, counters 0, delays 0, stop rows
    old = {k: v for k, v in sd.items() if not k.startswith("action_delay")}
    c = UpkieSim(n, model=model, config=_config())
    c.set_action_delay(2, 3)
    c.load_state_dict(old)
    assert c._action_delay is None
    count, delay, command = (x.cpu().numpy() for x in c.get_action_delay_state())
    assert not count.any() and not delay.any()
    assert np.all(np.isnan(command[:, :, 0])) and not command[:, :, 1:].any()


def test_rejections(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 64
    s = UpkieSim(n, model=model, config=_config())
    s.set_action_delay(1, 2)
    for low, high in ((3, 2), (0, 6)):
        with pytest.raises(UpkieRuntimeError):
            s.set_action_delay(low, high)
        assert s._action_delay == (1, 2)
    with pytest.raises(UpkieRuntimeError):
        UpkieSim(n, model=model, config=_config(joint_limits=0)).set_action_delay(0, 1)
    with pytest.raises(UpkieRuntimeError):
        UpkieSim(n, model=model, config=_config(spine_mode=1)).set_action_delay(0, 1)
    # set_config refuses fewer substeps than the range needs, and no joint limits
    with pytest.raises(UpkieRuntimeError):
        s.set_config(_config(nb_substeps=1))
    with pytest.raises(UpkieRuntimeError):
        s.set_config(_config(joint_limits=0))
    s.set_config(_config(nb_substeps=2))
    # the in-kernel rollout transports
    m = UpkieSim(64, model=model, config=_config(max_episode_steps=0))
    m.set_action_delay(0, 1)
    with pytest.raises(UpkieRuntimeError, match="action delay has no in-kernel rollout transport"):
        obs = torch.empty((64, 18), device="cuda")
        term = torch.empty(64, dtype=torch.uint8, device="cuda")
        m.step_servos_peers(_action(torch, model, "servos", 64, 0), [obs.data_ptr()], [term.data_ptr()])


def test_none_returns_to_the_old_families(model, torch):
    n, T = 256, 30
    cfg = _config()
    sim = _sim(model, cfg, n, 1, (2, 5), table=True)
    twin = _sim(model, cfg, n, 1, table=True)
    sim.set_action_delay(None)
    sim.set_state(twin.get_state())
    for k in range(T):
        x = _step(sim, "servos", _action(torch, model, "servos", n, k))
        y = _step(twin, "servos", _action(torch, model, "servos", n, k))
        for u, v in zip(x, y):
            assert _bits(u) == _bits(v), k


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import neutral_action

    n = 128
    env = B200VectorEnv(n, env_type, autoreset_mode="next_step", max_episode_steps=25, action_delay=(0.001, 0.004))
    assert env.sim._action_delay == (1, 4)  # 1 ms substeps at 200 Hz
    dim = {"servos": None, "gyropod": 2, "pendulum": 1, "base_velocity": 2}[env_type]
    gen = torch.Generator(device="cuda")

    def run():
        env.reset(seed=5)
        count, delay, _ = (x.cpu().numpy() for x in env.sim.get_action_delay_state())
        assert np.all(count == 1)
        np.testing.assert_array_equal(delay.astype(np.uint32),
                                      action_delay_draw_np(1, 4, 5, np.arange(n, dtype=np.uint64), 1))
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
        return out

    first, second = run(), run()
    for x, y in zip(first, second):
        for u, v in zip(x, y):
            assert torch.equal(torch.nan_to_num(u, nan=1e30), torch.nan_to_num(v, nan=1e30))
    env.set_action_delay(None)
    assert env.sim._action_delay is None
    with pytest.raises(UpkieException):
        env.set_action_delay(0.006)  # more than one 5 ms tick
    env.close()
