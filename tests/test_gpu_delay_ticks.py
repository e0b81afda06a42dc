# SPDX-License-Identifier: Apache-2.0
"""Delays of more than one tick on the device (upkie_b200_set_action_delay_ticks / set_observation_delay_ticks): a
deeper history changes nothing while the delays stay within one tick, a delay of q ticks and r substeps is the delay r
fed (action) or read (observation) q ticks late, clamped at each env's reset, checkpoints and depth changes keep the
history in age order, the rejections, and the vector envs at 1 kHz."""
import numpy as np
import pytest
import torch as torch_mod

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_gpu_action_delay import SEED, _action, _bits, _config, _step

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _sim(model, cfg, n, mode, action=None, sense=None, ticks=1, table=False, env_offset=0):
    """a handle with the delays set at depth `ticks`, then reset once (the explicit reset draws every env's delays)"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if table:
        s.set_env_params(s.get_env_params())
    if action is not None:
        s.set_action_delay(*action, max_ticks=ticks)
    if sense is not None:
        s.set_observation_delay(*sense, max_ticks=ticks)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


# ---- 1. the depth does not matter while the delays stay within one tick -------------------------------------------------


@pytest.mark.parametrize("which", ["action", "observation", "action_body"])
@pytest.mark.parametrize("path", ["device", "host"])
@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_depth_unused_changes_nothing(model, torch, kind, mode, path, which):
    if path == "host" and kind == "pendulum":
        pytest.skip("the host-buffer path steps UpkieServos and UpkieGyropod")
    n, T = 512, 70
    cfg = _config(body_contacts=1 if which == "action_body" else 0)
    nb = cfg.nb_substeps
    kw = {"sense": (0, nb)} if which == "observation" else {"action": (0, nb)}
    deep = _sim(model, cfg, n, mode, ticks=4, **kw)
    flat = _sim(model, cfg, n, mode, ticks=1, **kw)
    # The depth-4 handle runs the k_step_hist copy of its family. As test_gpu_action_delay.py's zero-delay test finds
    # for the host-buffer (TILE=1) copies of two families, separately compiled copies of the same physics can differ in
    # the last bits of an fp32 result (here the gyropod observation recomputed from the sensed state); on the host path
    # the twin is put back on the deep handle's state before every tick, integer outputs compared bit for bit and
    # observations within fp32 round-off of one tick.
    resync = path == "host"
    resets = 0
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        if resync:
            flat.set_state(deep.get_state())
            torch.cuda.synchronize()
        out_d = _step(deep, kind, a, path)
        out_f = _step(flat, kind, a, path)
        for x, y in zip(out_d, out_f):
            if resync and x.dtype == np.float32:
                np.testing.assert_allclose(x, y, rtol=1e-5, atol=1e-3, err_msg=str(k))
            else:
                assert _bits(x) == _bits(y), k
        resets += int(((out_d[2] != 0) | (out_d[3] != 0)).sum())
    if not resync:
        assert _bits(deep.get_state().cpu().numpy()) == _bits(flat.get_state().cpu().numpy())
    if kind == "servos" and which == "observation" and not resync:
        assert _bits(deep.spine_obs().cpu().numpy()) == _bits(flat.spine_obs().cpu().numpy())
    assert resets > 0


# ---- 2. the action delay of q ticks and r substeps is the delay r fed q ticks late ---------------------------------------


@pytest.mark.parametrize("nb, d", [(5, 7), (5, 10), (5, 13), (5, 20), (1, 2), (1, 4)])
def test_action_shift_oracle(model, torch, nb, d):
    from upkie_b200.sim import stop_commands

    n, T, K = 512, 110, 4
    q, r = divmod(d, nb)
    cfg = _config(nb_substeps=nb, max_episode_steps=30)
    a_sim = _sim(model, cfg, n, 1, action=(d, d), ticks=K)  # next-step auto-reset
    b_sim = _sim(model, cfg, n, 1, action=(r, r))
    stop = stop_commands(n, "cuda")
    acts, last_reset = [], torch.full((n,), -1, dtype=torch.int64, device="cuda")
    resetting = torch.zeros(n, dtype=torch.bool, device="cuda")
    resets = 0
    for t in range(T):
        last_reset = torch.where(resetting, torch.full_like(last_reset, t), last_reset)
        acts.append(_action(torch, model, "servos", n, t))
        if t - q >= 0:
            late = torch.where((last_reset < t - q)[:, None, None], acts[t - q], stop)
        else:
            late = stop
        out_a = _step(a_sim, "servos", acts[t])
        out_b = _step(b_sim, "servos", late.contiguous())
        for x, y in zip(out_a, out_b):
            assert _bits(x) == _bits(y), t
        done = (out_a[2] != 0) | (out_a[3] != 0)
        resets += int(done.sum())
        resetting = torch.from_numpy(done).to("cuda")
    assert _bits(a_sim.get_state().cpu().numpy()) == _bits(b_sim.get_state().cpu().numpy())
    assert resets > 0  # the run crossed fused resets


# ---- 3. the observation delay of q ticks and r substeps is the delay r read q ticks late ---------------------------------


SENSED_COLS = {"servos": None, "gyropod": [0, 1, 3, 4], "pendulum": None}  # gyropod 2, 5: the wrapper's yaw, undelayed


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
@pytest.mark.parametrize("nb, d", [(5, 8), (5, 10), (5, 13), (5, 20), (1, 3)])
def test_observation_shift_oracle(model, torch, kind, mode, nb, d):
    """The reports of a delay d = q nb + r handle equal those of a delay r twin q ticks earlier, bit for bit, clamped to
    the reset's observation after each reset: observations, spine observations, and in same-step mode the terminal
    step's final_obs and final spine observation. The gyropod wrapper's yaw columns match the twin at the same tick."""
    from test_gpu_observation_delay import _step as _step_fin

    n, T, K = 512, 100, 4
    q = (d - 1) // nb  # d = q * nb + r with 1 <= r <= nb (include/upkie_b200.h): r = nb snapshots the start of a tick
    r = d - q * nb
    same = mode == 2
    cfg = _config(nb_substeps=nb, max_episode_steps=30)
    a_sim = _sim(model, cfg, n, mode, sense=(d, d), ticks=K)
    b_sim = _sim(model, cfg, n, mode, sense=(r, r))
    cols = SENSED_COLS[kind] or slice(None)
    obs_b, spine_b = [], []
    last_reset = np.full(n, -10**6)  # the last tick whose step returned a post-reset observation, before this one
    pending = np.zeros(n, dtype=bool)  # next-step mode: the envs this step resets
    checked = finals = 0
    idx = np.arange(n)
    for t in range(T):
        if not same:
            last_reset[pending] = t
        a = _action(torch, model, kind, n, t)
        out_a = _step_fin(a_sim, kind, a, same_step=same)
        out_b = _step_fin(b_sim, kind, a, same_step=same)
        for x, y in zip(out_a[1:3], out_b[1:3]):  # the physics does not depend on the delay
            assert _bits(x) == _bits(y), t
        obs_b.append(out_b[0])
        spine_b.append(out_b[5])
        done = (out_a[1] | out_a[2]).astype(bool)
        src = np.maximum(t - q, last_reset)  # the report of tick t - q, or the reset's
        ok = src >= 0
        fin = same & done  # same-step resets: the terminal report is final_obs; the step returns the reset's
        cur = ok & ~fin
        s_src = np.where(ok, src, t)
        want = np.stack([obs_b[s][i] for i, s in zip(idx, s_src)])
        assert _bits(out_a[0][cur][:, cols]) == _bits(want[cur][:, cols]), t
        assert _bits(out_a[0][fin]) == _bits(out_b[0][fin]), t  # the post-reset observation, undelayed
        if kind == "gyropod":
            assert _bits(out_a[0][:, [2, 5]]) == _bits(out_b[0][:, [2, 5]]), t
        if kind == "servos":
            want_s = np.stack([spine_b[s][i] for i, s in zip(idx, s_src)])
            assert _bits(out_a[5][cur]) == _bits(want_s[cur]), t
        if fin.any():
            sel = fin & ok
            assert _bits(out_a[3][sel][:, cols]) == _bits(want[sel][:, cols]), t
            if kind == "gyropod":
                assert _bits(out_a[3][fin][:, [2, 5]]) == _bits(out_b[3][fin][:, [2, 5]]), t
            if kind == "servos":
                assert _bits(out_a[4][sel]) == _bits(want_s[sel]), t
            finals += int(sel.sum())
            last_reset[fin] = t
        checked += int(ok.sum())
        pending = done
    assert checked > n * (T - q - 1) // 2 and (last_reset > 0).any()
    if same:
        assert finals > 0  # terminal steps observed under the history


# ---- 4. the draws over the widened range -------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "pendulum"])
@pytest.mark.parametrize("mode", [1, 2])
def test_draws_follow_the_law(model, torch, kind, mode):
    from test_action_delay_cpu import action_delay_draw_np
    from test_observation_delay_cpu import observation_delay_draw_np

    n, T, K = 1024, 150, 4
    cfg = _config()
    high = K * cfg.nb_substeps
    sim = _sim(model, cfg, n, mode, action=(0, high), sense=(1, high), ticks=K)
    g = np.arange(n, dtype=np.uint64)
    expect = np.ones(n, dtype=np.uint64)  # the explicit reset after the specs: draw 1

    def check():
        count, delay, _ = (x.cpu().numpy() for x in sim.get_action_delay_state())
        np.testing.assert_array_equal(count.astype(np.uint64), expect)
        np.testing.assert_array_equal(delay.astype(np.uint32), action_delay_draw_np(0, high, SEED, g, expect))
        count, delay, _ = (x.cpu().numpy() for x in sim.get_observation_delay_state())
        np.testing.assert_array_equal(count.astype(np.uint64), expect)
        np.testing.assert_array_equal(delay.astype(np.uint32), observation_delay_draw_np(1, high, SEED, g, expect))
        return delay

    done_prev = np.zeros(n, dtype=bool)
    for k in range(T):
        out = _step(sim, kind, _action(torch, model, kind, n, k))
        done = (out[2] | out[3]).astype(bool)
        expect += (done_prev if mode == 1 else done).astype(np.uint64)
        done_prev = done
    delay = check()
    assert expect.max() > 3 and delay.max() > cfg.nb_substeps  # draws beyond one tick
    # explicit masked resets, with device-sampled and with host rows: the whole history is refilled
    for init in (None, "host"):
        mask = ((np.arange(n) % 3) == (0 if init is None else 1)).astype(np.uint8)
        rows = None
        if init == "host":
            rows = torch.zeros((n, _abi.INIT_DIM), device="cuda")
            rows[:, 2] = 0.58
            rows[:, 3] = 1.0
        sim.reset(mask=torch.from_numpy(mask).cuda(), init_state=rows, seed=SEED)
        expect = expect + mask.astype(np.uint64)
        check()
        sel = mask == 1
        cmd = sim.get_action_delay_history().cpu().numpy()[:, sel]
        assert np.all(np.isnan(cmd[..., 0])) and not cmd[..., 1:].any()
        snaps = sim.get_observation_delay_history().cpu().numpy()[:, sel]
        state = sim.get_state().cpu().numpy()[sel]
        for a in range(K):
            assert _bits(snaps[a]) == _bits(state)


def test_shards_reproduce_the_batch(model, torch):
    n, T, K = 1024, 80, 4
    cfg = _config()
    spec = {"action": (0, K * cfg.nb_substeps), "sense": (0, K * cfg.nb_substeps), "ticks": K}
    whole = _sim(model, cfg, n, 2, **spec)
    half = n // 2
    shards = [_sim(model, cfg, half, 2, env_offset=o, **spec) for o in (0, half)]
    for k in range(T):
        out = _step(whole, "servos", _action(torch, model, "servos", n, k))
        for s, o in zip(shards, (0, half)):
            part = _step(s, "servos", _action(torch, model, "servos", half, k, env_offset=o, total=n))
            for x, y in zip(part, out):
                assert _bits(x) == _bits(y[o : o + half]), k
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_action_delay_state() + s.get_observation_delay_state(),
                        whole.get_action_delay_state() + whole.get_observation_delay_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o : o + half])
        assert _bits(s.get_action_delay_history().cpu().numpy()) == \
            _bits(whole.get_action_delay_history().cpu().numpy()[:, o : o + half])
        assert _bits(s.get_observation_delay_history().cpu().numpy()) == \
            _bits(whole.get_observation_delay_history().cpu().numpy()[:, o : o + half])


# ---- 5. checkpoints and depth changes --------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    n, K = 256, 4
    cfg = _config()
    nb = cfg.nb_substeps
    sim = _sim(model, cfg, n, 1, action=(0, K * nb), sense=(0, K * nb), ticks=K)
    for k in range(15):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    sd = sim.state_dict()
    assert sd["action_delay_ticks"] == K and sd["observation_delay_ticks"] == K
    assert tuple(sd["action_delay_history"].shape) == (K, n, 6, 6)
    fresh = _sim(model, cfg, n, 0)
    fresh.load_state_dict(sd)
    torch.cuda.synchronize()
    for k in range(15, 40):
        a = _action(torch, model, "servos", n, k)
        for x, y in zip(_step(sim, "servos", a), _step(fresh, "servos", a)):
            assert _bits(x) == _bits(y), k
    assert _bits(sim.get_state().cpu().numpy()) == _bits(fresh.get_state().cpu().numpy())


def test_checkpoint_of_a_delay_turned_off_keeps_its_history(model, torch):
    """A handle whose delays are off keeps its depth-4 histories; a checkpoint carries them, so that turning the delays
    on again continues alike on the handle and on its restored copy"""
    n, K = 256, 4
    cfg = _config()
    nb = cfg.nb_substeps
    sim = _sim(model, cfg, n, 1, action=(0, K * nb), sense=(0, K * nb), ticks=K)
    for k in range(12):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    sim.set_action_delay(None)
    sim.set_observation_delay(None)
    sd = sim.state_dict()
    assert sd["action_delay"] is None and sd["action_delay_ticks"] == K and sd["observation_delay_ticks"] == K
    fresh = _sim(model, cfg, n, 0)
    fresh.load_state_dict(sd)
    for h in (sim, fresh):
        h.set_action_delay(0, K * nb, max_ticks=K)
        h.set_observation_delay(0, K * nb, max_ticks=K)
    assert _bits(fresh.get_action_delay_history().cpu().numpy()) == _bits(sim.get_action_delay_history().cpu().numpy())
    torch.cuda.synchronize()
    for k in range(12, 30):
        a = _action(torch, model, "servos", n, k)
        for x, y in zip(_step(sim, "servos", a), _step(fresh, "servos", a)):
            assert _bits(x) == _bits(y), k


def test_depth_change_keeps_age_order(model, torch):
    from upkie_b200.sim import stop_commands

    n, nb = 128, 5
    cfg = _config(max_episode_steps=0, servos_fall_termination=0)
    sim = _sim(model, cfg, n, 0, action=(0, 4 * nb), sense=(0, 4 * nb), ticks=4)
    for k in range(6):
        _step(sim, "servos", _action(torch, model, "servos", n, k))
    cmd4 = sim.get_action_delay_history().cpu()
    snap4 = sim.get_observation_delay_history().cpu()
    assert _bits(cmd4[0].numpy()) == _bits(sim.get_action_delay_state()[2].cpu().numpy())  # the previous tick's
    assert not torch.isnan(cmd4[:, :, :, 0]).any()  # six ticks filled all four commands: no stop row is left
    sim.set_action_delay(0, 6 * nb, max_ticks=6)
    sim.set_observation_delay(0, 6 * nb, max_ticks=6)
    cmd6, snap6 = sim.get_action_delay_history().cpu(), sim.get_observation_delay_history().cpu()
    assert _bits(cmd6[:4].numpy()) == _bits(cmd4.numpy())
    assert _bits(cmd6[4:].nan_to_num(7.0).numpy()) == _bits(stop_commands(n).expand(2, n, 6, 6).nan_to_num(7.0).numpy())
    assert _bits(snap6[:4].numpy()) == _bits(snap4.numpy())
    assert _bits(snap6[4].numpy()) == _bits(snap4[3].numpy()) and _bits(snap6[5].numpy()) == _bits(snap4[3].numpy())
    sim.set_action_delay(0, 2 * nb, max_ticks=2)
    sim.set_observation_delay(0, 2 * nb, max_ticks=2)
    assert _bits(sim.get_action_delay_history().cpu().numpy()) == _bits(cmd4[:2].numpy())
    assert _bits(sim.get_observation_delay_history().cpu().numpy()) == _bits(snap4[:2].numpy())
    sim.set_action_delay(0, nb)
    assert _bits(sim.get_action_delay_state()[2].cpu().numpy()) == _bits(cmd4[0].numpy())
    # a reset fills the whole history
    sim.set_action_delay(0, 4 * nb, max_ticks=4)
    sim.reset(seed=SEED)
    h = sim.get_action_delay_history()
    assert _bits(h.nan_to_num(7.0).cpu().numpy()) == _bits(stop_commands(n, "cuda").expand(4, n, 6, 6).nan_to_num(7.0)
                                                           .cpu().numpy())


# ---- 6. rejections and the vector envs ------------------------------------------------------------------------------


def test_rejections(model, torch):
    cfg = _config()
    nb = cfg.nb_substeps
    sim = _sim(model, cfg, 64, 1)
    for setter in (sim.set_action_delay, sim.set_observation_delay):
        for bad in (0, _abi.MAX_DELAY_TICKS + 1):
            with pytest.raises(UpkieRuntimeError, match="max_ticks outside"):
                setter(0, 1, max_ticks=bad)
        with pytest.raises(UpkieRuntimeError, match="max_ticks \\* nb_substeps"):
            setter(0, 3 * nb + 1, max_ticks=3)
        with pytest.raises(UpkieRuntimeError, match="at most one tick"):
            setter(0, nb + 1)
    sim.set_action_delay(0, 3 * nb, max_ticks=3)
    assert sim._action_delay == (0, 3 * nb)
    sim.set_observation_delay(0, 2 * nb + 1, max_ticks=3)
    small = _config(nb_substeps=nb - 1)  # ceil(15 / 3) = 5 > 4
    with pytest.raises(UpkieRuntimeError, match="nb_substeps below the action delay"):
        sim.set_config(small)
    sim.set_action_delay(0, 2 * nb, max_ticks=3)
    sim.set_config(_config(nb_substeps=nb - 1))  # 3 * 4 >= 11 and >= 10
    sim.set_action_delay(None)
    with pytest.raises(UpkieRuntimeError, match="nb_substeps below the observation delay"):
        sim.set_config(_config(nb_substeps=3))


@pytest.mark.parametrize("kind", ["servos", "pendulum"])
def test_none_returns_to_the_one_tick_kernels(model, torch, kind):
    """Turning both delays off on a depth-4 handle steps bit for bit like a handle that never had them (FAM_TABLE)"""
    n, T, K = 256, 30, 4
    cfg = _config(max_episode_steps=0, servos_fall_termination=0)  # no resets: the counters of the steps before agree
    nb = cfg.nb_substeps
    sim = _sim(model, cfg, n, 0, action=(2, K * nb), sense=(1, K * nb), ticks=K, table=True)
    twin = _sim(model, cfg, n, 0, table=True)
    for k in range(10):  # both handles step, so that their tick counters agree
        _step(sim, kind, _action(torch, model, kind, n, k))
        _step(twin, kind, _action(torch, model, kind, n, k))
    sim.set_action_delay(None)
    sim.set_observation_delay(None)
    sim.set_state(twin.get_state())
    torch.cuda.synchronize()
    for k in range(T):
        x = _step(sim, kind, _action(torch, model, kind, n, k))
        y = _step(twin, kind, _action(torch, model, kind, n, k))
        for u, v in zip(x, y):
            assert _bits(u) == _bits(v), k
    assert _bits(sim.spine_obs().cpu().numpy()) == _bits(twin.spine_obs().cpu().numpy())


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env_at_1khz(torch, env_type):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import neutral_action

    n = 128
    with pytest.raises(UpkieException, match="more than one tick"):
        B200VectorEnv(n, env_type, frequency=1000.0, action_delay=(0.001, 0.004))
    dim = {"servos": None, "gyropod": 2, "pendulum": 1, "base_velocity": 2}[env_type]
    gen = torch.Generator(device="cuda")

    def make():
        env = B200VectorEnv(n, env_type, frequency=1000.0, autoreset_mode="next_step", max_episode_steps=60,
                            max_delay_ticks=4, action_delay=(0.001, 0.004), observation_delay=0.003)
        assert env.config.nb_substeps == 1
        assert env.sim._action_delay == (1, 4) and env.sim._observation_delay == (3, 3)
        return env

    # Each run starts from a fresh env: the first ticks of an episode report its post-reset state, whose measured
    # torques a reset with host rows leaves as the state before the reset held them
    def run():
        nonlocal env
        env = make()
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
        return out

    env = None
    first = run()
    env.close()
    second = run()
    for (o1, t1, s1), (o2, t2, s2) in zip(first, second):
        assert torch.equal(t1, t2) and _bits(s1.cpu().numpy()) == _bits(s2.cpu().numpy())
        assert _bits(o1.cpu().numpy()) == _bits(o2.cpu().numpy())
    env.set_action_delay(None)
    env.set_observation_delay(None)
    assert env.sim._action_delay is None and env.sim._observation_delay is None
    env.reset(seed=5)
    env.step_tensors(neutral_action(env.model, n, "cuda") if dim is None else torch.zeros((n, dim), device="cuda"))
    env.set_action_delay(0.002)
    assert env.sim._action_delay == (2, 2) and env.sim._action_delay_ticks == 4
    env.close()
