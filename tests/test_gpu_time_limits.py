# SPDX-License-Identifier: Apache-2.0
"""Episode time limits in the step kernel (config.max_episode_steps): the truncation schedule in the three auto-reset
modes, the bookkeeping against a host-side TimeLimit model, the final observations of same-step auto-resets, the
vector env, checkpoints, shards, and the calls that reject a limit."""
import ctypes as C

import numpy as np
import pytest

from upkie_b200 import _abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _sim(n, model, cfg, mode, seed=7, env_offset=0):
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, seed, env_offset)
    s.reset(seed=seed, env_offset=env_offset)
    return s


def _headline_config(limit):
    """The headline workload's physics (bench.py servos_config): fall termination, random initial pitch."""
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.max_episode_steps = limit
    return cfg


def _torque_actions(torch, model, n, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    tau = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")

    def make():
        a = torch.zeros((n, 6, 6), device="cuda")
        a[:, :, 0] = float("nan")
        a[:, :, 5] = tau
        a[:, :, 2] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * tau
        return a

    return make


def _pendulum_policy(o):
    """README policy: keeps the pendulum envs up."""
    n = o.shape[0]
    return (10.0 * o[:, 0] + 1.0 * o[:, 1] + 0.0 * o[:, 2] + 0.1 * o[:, 3]).reshape(n, 1).astype(np.float32)


# ---- 1. exact schedule ----------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["same_step", "next_step", "disabled"])
def test_truncation_schedule(model, torch, mode):
    from upkie_b200.envs import B200VectorEnv

    n, T = 256, 50
    env = B200VectorEnv(n, "pendulum", model=model, autoreset_mode=mode, max_episode_steps=T)
    o, _ = env.reset(seed=0)
    if mode == "same_step":
        for k in range(1, 151):
            o, _, te, tr, info = env.step(_pendulum_policy(o))
            assert not te.any()
            assert tr.all() if k % T == 0 else not tr.any(), k
            assert ("final_obs" in info) == (k % T == 0)
            if k % T == 0:
                assert info["_final_obs"].all() and info["final_obs"].shape == (n, 4)
    elif mode == "next_step":
        truncated_at = {50, 101, 152}
        for k in range(1, 153):
            o, _, te, tr, info = env.step(_pendulum_policy(o))
            assert not te.any()
            assert tr.all() if k in truncated_at else not tr.any(), k
            assert "final_obs" not in info
            if k - 1 in truncated_at:  # the reset step: both flags 0 and the reset observation
                assert np.array_equal(o, env.sim.reset_obs(4).cpu().numpy())
                assert np.abs(o[:, 0]).max() < 1e-2
    else:
        for k in range(1, 61):
            o, _, te, tr, _ = env.step(_pendulum_policy(o))
            assert tr.all() if k >= T else not tr.any(), k
        mask = np.zeros(n, np.uint8)
        mask[::2] = 1
        o, _ = env.reset(options={"reset_mask": mask})
        for k in range(61, 116):
            o, _, te, tr, _ = env.step(_pendulum_policy(o))
            assert tr[1::2].all(), k  # not reset: truncated until the user resets them
            assert tr[::2].all() if k >= 60 + T else not tr[::2].any(), k
    env.close()


# ---- 2. mixed falls and time-outs: bit-exact bookkeeping ------------------------------------------------------------

def test_timelimit_bookkeeping_against_host_model(model, torch):
    n, T, steps = 65536, 40, 300
    a = _sim(n, model, _headline_config(T), 1)
    b = _sim(n, model, _headline_config(0), 1)  # twin without a limit: the same kernel, the limit is a runtime value
    act = _torque_actions(torch, model, n, 3)
    elapsed = np.zeros(n, np.int64)
    pending = np.zeros(n, bool)
    timed_out = torch.zeros(n, dtype=torch.bool, device="cuda")
    falls = timeouts = both = 0
    for k in range(steps):
        u = act()
        oa, ta, ra = a.step_servos_compact_truncated(u)
        ob, tb = b.step_servos_compact(u)
        # until its first time-out (that step included) every env matches the twin bit for bit
        live = ~timed_out
        assert torch.equal(oa[live], ob[live]) and torch.equal(ta[live], tb[live]), k
        term, trunc = ta.cpu().numpy().astype(bool), ra.cpu().numpy().astype(bool)
        # host-side TimeLimit fed the returned `terminated`; the next-step reset step is not counted
        elapsed = np.where(pending, 0, elapsed + 1)
        expect = ~pending & (elapsed >= T)
        assert np.array_equal(trunc, expect), (k, np.flatnonzero(trunc != expect)[:8])
        assert not term[pending].any()
        pending = term | trunc
        timed_out |= torch.from_numpy(trunc).cuda()
        falls += int((term & ~trunc).sum())
        timeouts += int((trunc & ~term).sum())
        both += int((term & trunc).sum())
    assert falls > 0 and timeouts > 0, (falls, timeouts, both)


# ---- 3. final observations of same-step auto-resets -----------------------------------------------------------------

SENTINEL = -12345.0


def _final_obs_case(torch, model, kind):
    """(config, n, step(sim, k, final_obs or None) -> (obs, terminated, truncated), final_obs buffer maker)."""
    n = 4096
    cfg = _headline_config(40)
    cfg.rand_pitch = 0.6  # some robots fall before their first time-out
    gen = torch.Generator(device="cuda")
    if kind in ("servos", "compact", "host_compact", "spine"):
        if kind == "spine":
            cfg.spine_mode = 1
        acts = [_torque_actions(torch, model, n, 11 + j)() for j in range(4)]

        if kind in ("servos", "spine"):
            def step(s, k, fin):
                o, _, t, r = s.step_servos(acts[k % 4], final_obs=fin)
                return o, t, r
            shape = (n, 6, 5)
        elif kind == "compact":
            def step(s, k, fin):
                return s.step_servos_compact_truncated(acts[k % 4], final_obs=fin)
            shape = (n, 6, 3)
        else:
            host = [x.cpu().numpy() for x in acts]

            def step(s, k, fin):
                o, t, r, f = s.step_host(host[k % 4], 36, compact=True, final_obs=fin is not None)
                if fin is not None:
                    fin[:] = torch.from_numpy(f)
                return torch.from_numpy(o.copy()), torch.from_numpy(t.copy()), torch.from_numpy(r.copy())
            shape = (n, 6, 3)
    else:
        # full ground velocity, one direction per env: the robots that do not fall within the limit time out
        cfg.max_episode_steps = 80
        dim = 2 if kind == "gyropod" else 1
        gen.manual_seed(5)
        sign = torch.where(torch.rand((n, dim), device="cuda", generator=gen) < 0.5, -1.0, 1.0)
        acts = [(3.0 * sign).contiguous()] * 4
        fn = "step_gyropod" if kind == "gyropod" else "step_pendulum"

        def step(s, k, fin):
            o, _, t, r = getattr(s, fn)(acts[k % 4], final_obs=fin)
            return o, t, r
        shape = (n, 6) if kind == "gyropod" else (n, 4)
    return cfg, n, step, shape


@pytest.mark.parametrize("kind", ["servos", "compact", "host_compact", "gyropod", "pendulum", "spine"])
def test_final_obs_equals_the_twin_without_autoreset(model, torch, kind):
    """Servo rows are bit-identical to the twin's. The gyropod / pendulum kernels of the two auto-reset modes are
    compiled apart and already differ from the twin at fp32 round-off after one step: there the rows are compared to
    that round-off."""
    cfg, n, step, shape = _final_obs_case(torch, model, kind)
    exact = kind not in ("gyropod", "pendulum")

    def same(x, y):
        return torch.equal(x, y) if exact else bool(((x - y).abs() <= 1e-5 + 1e-4 * y.abs()).all())

    a = _sim(n, model, cfg, 2)
    b = _sim(n, model, cfg, 0)  # auto-reset disabled: returns the observation the resetting envs reached
    if kind == "host_compact":
        a._host_final_obs(18)  # the pinned rows the kernel stores into
    fin = torch.empty(shape, dtype=torch.float32, device="cuda" if kind != "host_compact" else "cpu")
    first = torch.zeros(n, dtype=torch.bool)  # env has reset once: from there on it differs from the twin
    reasons = set()
    for k in range(2 * cfg.max_episode_steps + 20):
        fin.fill_(SENTINEL)
        if kind == "host_compact":
            a._host_final_obs(18)[:] = SENTINEL
        oa, ta, ra = step(a, k, fin)
        ob, tb, rb = step(b, k, None)
        oa, ta, ra, ob, fa = oa.cpu(), ta.cpu().bool(), ra.cpu().bool(), ob.cpu(), fin.cpu()
        reset = ta | ra
        fresh = reset & ~first
        live = ~first
        assert torch.equal(ta[live], tb.cpu().bool()[live]), k
        assert same(fa[fresh], ob[fresh]), (kind, k)  # the terminal rows the twin returns
        assert (fa[~reset] == SENTINEL).all(), (kind, k)  # rows of the other envs are untouched
        if fresh.any():
            reasons |= {"fall"} if (ta & fresh).any() else set()
            reasons |= {"time-out"} if (ra & ~ta & fresh).any() else set()
        assert same(oa[live & ~reset], ob[live & ~reset]), k
        first |= reset
    assert first.all() and reasons == {"fall", "time-out"}, (int(first.sum()), reasons)


# ---- 4. vector env: host arrays and device tensors agree -------------------------------------------------------------

@pytest.mark.parametrize("copy", [True, False])
@pytest.mark.parametrize("env_type", ["servos", "pendulum"])
def test_vector_env_final_obs_host_and_tensors(model, torch, env_type, copy):
    """The host path runs the shared-memory-tile kernels, step_tensors the device-buffer ones: flags and masks agree
    exactly, observations to fp32 round-off (as for the plain steps, test_gpu_envs.py). The actions keep every robot
    up, so every reset is a time-out."""
    from upkie_b200.envs import B200VectorEnv

    # servos: no balance control, so a short limit keeps the compared states close to the upright start
    n, T = 512, (4 if env_type == "servos" else 20)
    kw = dict(model=model, autoreset_mode="same_step", max_episode_steps=T, copy=copy)
    host = B200VectorEnv(n, env_type, **kw)
    dev = B200VectorEnv(n, env_type, **kw)
    o, _ = host.reset(seed=1)
    dev.reset(seed=1)
    seen = 0
    for k in range(1, 2 * T + 3):
        if env_type == "servos":
            act = np.zeros((n, 6, 6), np.float32)
            act[:, :, 0] = np.nan
            act[:, :, 3] = act[:, :, 4] = 1.0
            act[:, :, 5] = np.asarray(model.tau_max, np.float32)
        else:
            act = _pendulum_policy(o)
        o, _, te, tr, info = host.step(act)
        do, _, dte, dtr, dinfo = dev.step_tensors(torch.from_numpy(act).cuda())
        assert np.array_equal(te, dte.cpu().numpy().astype(bool)) and np.array_equal(tr, dtr.cpu().numpy().astype(bool))
        assert ("final_obs" in info) == ("final_obs" in dinfo) == (k % T == 0), k
        if "final_obs" not in info:
            continue
        seen += 1
        mask = info["_final_obs"]
        assert mask.dtype == np.bool_ and np.array_equal(mask, dinfo["_final_obs"].cpu().numpy()) and mask.all()
        dfin = dinfo["final_obs"].cpu().numpy()
        if env_type == "servos":
            fin = np.stack([np.concatenate([info["final_obs"][j][key] for key in _abi.OBS_KEYS], axis=1)
                            for j in _abi.JOINT_NAMES], axis=1)
        else:
            fin = info["final_obs"]
        d = np.abs(fin[mask] - dfin[mask])
        assert d.max() < 2e-2 and np.median(d) < 1e-5, (d.max(), np.median(d))
        if copy:  # copies survive the next step
            keep = np.array(fin, copy=True)
            host.step(act)
            after = info["final_obs"] if env_type != "servos" else info["final_obs"]["left_hip"]["position"]
            before = keep if env_type != "servos" else keep[:, 0, 0:1]
            assert np.array_equal(after, before)
            dev.step_tensors(torch.from_numpy(act).cuda())
            break
    assert seen >= 1
    host.close()
    dev.close()


# ---- 5. checkpoints and shards ----------------------------------------------------------------------------------------

def test_checkpoint_continues_bit_for_bit(model, torch):
    n = 4096
    a = _sim(n, model, _headline_config(25), 1)
    act = _torque_actions(torch, model, n, 21)
    acts = [act() for _ in range(70)]
    for k in range(30):
        a.step_servos_compact_truncated(acts[k])
    sd = a.state_dict()
    assert sd["elapsed"].max() > 0
    b = _sim(n, model, _headline_config(25), 0)
    b.load_state_dict(sd)
    for k in range(30, 70):
        oa, ta, ra = a.step_servos_compact_truncated(acts[k])
        ob, tb, rb = b.step_servos_compact_truncated(acts[k])
        assert torch.equal(oa, ob) and torch.equal(ta, tb) and torch.equal(ra, rb), k
    # a checkpoint without the counts loads them as zeros
    sd = a.state_dict()
    del sd["elapsed"]
    b.load_state_dict(sd)
    assert int(b.state_dict()["elapsed"].abs().max()) == 0


def test_two_shards_reproduce_one_batch(model, torch):
    n = 2048
    act = _torque_actions(torch, model, 2 * n, 31)
    acts = [act() for _ in range(90)]
    whole = _sim(2 * n, model, _headline_config(30), 1, seed=9)
    shards = [_sim(n, model, _headline_config(30), 1, seed=9, env_offset=r * n) for r in range(2)]
    any_trunc = False
    for k in range(90):
        o, t, r = whole.step_servos_compact_truncated(acts[k])
        o, t, r = o.clone(), t.clone(), r.clone()
        for s, sl in zip(shards, (slice(0, n), slice(n, 2 * n))):
            so, st, sr = s.step_servos_compact_truncated(acts[k][sl].contiguous())
            assert torch.equal(so, o[sl]) and torch.equal(st, t[sl]) and torch.equal(sr, r[sl]), k
        any_trunc |= bool(r.any())
    assert any_trunc


# ---- 6. calls that reject a limit, base_velocity -----------------------------------------------------------------------

def test_in_kernel_transports_reject_a_limit(model, torch):
    from upkie_b200._lib import lib

    n = 64
    s = _sim(n, model, _headline_config(10), 1)
    action = torch.zeros((n, 6, 6), device="cuda")
    obs = torch.zeros((n, 6, 3), device="cuda")
    term = torch.zeros(n, dtype=torch.uint8, device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    launches = s.launches
    assert lib().upkie_b200_step_servos_multicast(s._h, p(action), p(obs), p(term), None) == -1
    assert b"max_episode_steps" in lib().upkie_b200_last_error()
    oa = (C.c_void_p * 1)(obs.data_ptr())
    ta = (C.c_void_p * 1)(term.data_ptr())
    assert lib().upkie_b200_step_servos_peers(s._h, p(action), oa, ta, 1, None) == -1
    assert lib().upkie_b200_step_servos_push(s._h, p(action), p(obs), p(term), None, None) == -1
    assert s.launches == launches  # nothing was launched


def test_base_velocity_reports_truncated(model, torch):
    from upkie_b200.envs import B200VectorEnv

    n, T = 64, 12
    env = B200VectorEnv(n, "base_velocity", model=model, max_episode_steps=T)
    env.reset(seed=0)
    for k in range(1, T + 3):
        _, _, te, tr, _ = env.step(np.zeros((n, 2), np.float32))
        assert not te.any()
        assert tr.all() if k >= T else not tr.any(), k
    env.close()
