# SPDX-License-Identifier: Apache-2.0
"""UpkieBaseVelocity vector envs with the fused epilogue (k_base_velocity_post) on the GPU: disabled mode gives the
bits of the torch epilogue, both auto-reset modes against a twin that a Gymnasium-style loop resets by mask, the golden
runs of the reference's own class, host arrays against tensors, shards, explicit resets, and the C entry's argument
checks."""
import ctypes as C
import json
import os

import numpy as np
import pytest

from upkie_b200 import _abi

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0
GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "base_velocity_autoreset_runs.json")


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _env(model, n, mode="disabled", **kw):
    from upkie_b200.envs import B200VectorEnv

    return B200VectorEnv(n, "base_velocity", model=model, autoreset_mode=mode, **kw)


def _ulp_distance(torch, a, b):
    """Largest distance in units in the last place between two float32 tensors (0 = identical bits)."""
    ia = a.contiguous().view(torch.int32).to(torch.int64)
    ib = b.contiguous().view(torch.int32).to(torch.int64)
    ia = torch.where(ia < 0, -(ia & 0x7FFFFFFF), ia)
    ib = torch.where(ib < 0, -(ib & 0x7FFFFFFF), ib)
    return int((ia - ib).abs().max())


# ---- 1. disabled mode: the bits of the parent's torch epilogue ------------------------------------------------------

def test_disabled_mode_equals_the_torch_epilogue(model, torch):
    """300 ticks at 4 096 envs with random actions: the fused path and base_velocity_tick (twin handles, same seed)
    give identical observations, flags and commanded velocities. The dead reckoning runs libdevice's cosf / sinf
    (base_velocity.cu is built without fast-math) against torch's CUDA cos / sin: the same IEEE routines."""
    from upkie_b200.base_velocity import base_velocity_tick

    n = 4096
    a, b = _env(model, n), _env(model, n)
    a.reset(seed=4)
    b.reset(seed=4)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(11)
    # yaw is never wrapped (upkie_gyropod.py:383-384): start the envs at |yaw| up to 60 rad, where approximate sin /
    # cos would lose accuracy, on both handles
    st = a.sim.get_state()
    st[:, _abi.ST_YAW] += (torch.rand(n, device="cuda", generator=gen) * 2 - 1) * 60.0
    a.sim.set_state(st.contiguous())
    b.sim.set_state(st.clone().contiguous())
    worst = 0
    for k in range(300):
        act = torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1
        oa, ra, ta, tra, _ = a.step_tensors(act)
        ob, rb, tb, trb, b._spine = base_velocity_tick(act, b._spine, b._xy, b.dt, b.mpc_balancer.step_spine,
                                                       b.sim.step_gyropod, b.sim.spine_obs)
        worst = max(worst, _ulp_distance(torch, oa, ob))
        assert torch.equal(ta, tb) and torch.equal(tra, trb) and torch.equal(ra, rb), k
        assert torch.equal(a.mpc_balancer.commanded_velocity, b.mpc_balancer.commanded_velocity), k
        assert torch.equal(a._xy, b._xy), k
    assert worst == 0, f"largest difference: {worst} ulp"
    assert float(oa[:, 2].abs().max()) > 50.0
    a.close()
    b.close()


# ---- 2. both auto-reset modes against a twin without auto-reset -----------------------------------------------------

def _push_half(env, n):
    from upkie_b200 import ExternalForce

    rng = np.random.default_rng(3)
    push = np.zeros((n, 3))
    push[::2, 0] = rng.uniform(20.0, 200.0, n)[::2]  # half the envs: forward pushes of many sizes, some fall
    env.set_external_forces({"torso": ExternalForce(push)})


@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_autoreset_equals_the_twin_without_autoreset(model, torch, mode):
    """Up to each env's first reset (that step included) flags agree exactly and observations to the fp32 round-off
    of the gyropod kernels of the two modes, which are compiled apart; the final observations are the twin's terminal
    [x, y, yaw]; reset envs show [0, 0, 0], x = y = 0 and commanded velocity 0; other final rows keep a sentinel."""
    n, T = 4096, 80
    a, b = _env(model, n, mode, max_episode_steps=T), _env(model, n, "disabled", max_episode_steps=T)
    for e in (a, b):
        e.reset(seed=2)
        _push_half(e, n)

    def same(x, y):
        return bool(((x - y).abs() <= 1e-5 + 1e-4 * y.abs()).all())

    act = torch.tensor([[0.3, 0.5]], device="cuda").repeat(n, 1).contiguous()
    first = torch.zeros(n, dtype=torch.bool)
    pending = torch.zeros(n, dtype=torch.bool)  # next_step: envs whose reset step is this one
    reasons = set()
    for k in range(2 * T + 20):
        if mode == "same_step":
            a._device_final_obs().fill_(SENTINEL)
        oa, _, ta, ra, info = a.step_tensors(act)
        ob, _, tb, rb, _ = b.step_tensors(act)
        oa, ta, ra, ob, tb, rb = oa.cpu(), ta.cpu().bool(), ra.cpu().bool(), ob.cpu(), tb.cpu().bool(), rb.cpu().bool()
        xy, vc = a._xy.cpu(), a.mpc_balancer.commanded_velocity.cpu()
        ended = ta | ra
        live = ~first & ~pending
        assert torch.equal(ta[live], tb[live]) and torch.equal(ra[live], rb[live]), k
        if mode == "same_step":
            fin = a._device_final_obs().cpu()
            assert (fin[~ended] == SENTINEL).all(), k
            fresh = ended & live
            assert same(fin[fresh], ob[fresh]), k  # the terminal rows the twin returns
            assert ("final_obs" in info) == bool(ended.any()), k
            reset_now = ended
        else:
            reset_now = pending
            fresh = ended & live
            assert same(oa[fresh], ob[fresh]), k  # the step that ends: [x, y, yaw] with the flags set
            assert not (ta[pending] | ra[pending]).any(), k  # the reset step: both flags 0
        assert not oa[reset_now].any() and not xy[reset_now].any() and not vc[reset_now].any(), k
        ok = live & ~reset_now & ~ended
        assert same(oa[ok], ob[ok]), k
        if fresh.any():
            reasons |= {"fall"} if (ta & fresh).any() else set()
            reasons |= {"time-out"} if (ra & ~ta & fresh).any() else set()
        first |= pending if mode == "next_step" else ended
        pending = ended if mode == "next_step" else pending
        # the twin: a Gymnasium-style loop that resets its ended envs by mask
        done = (tb | rb).numpy()
        if done.any():
            b.reset(options={"reset_mask": done})
    assert first.all() and reasons == {"fall", "time-out"}, (int(first.sum()), reasons)
    a.close()
    b.close()


# ---- 3. golden runs of the reference's own class --------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_autoreset_replays_the_reference_runs(model, torch, mode):
    from upkie_b200.robot_state import RobotState

    runs = json.load(open(GOLDEN))
    run, T = runs[mode], runs["time_limit"]
    n = 32  # identical copies: the batch stays identical too
    env = _env(model, n, mode, max_episode_steps=T,
               init_state=RobotState(position_base_in_world=np.array([0.0, 0.0, 0.58])))
    env.reset(seed=1)
    row = torch.tensor(run["init_row"], dtype=torch.float32, device="cuda").reshape(1, -1).repeat(n, 1).contiguous()
    env.sim.reset(init_state=row)
    env.mpc_balancer.reset()
    env._xy.zero_()
    env._spine = env.sim.spine_obs()
    worst_obs = worst_fin = worst_v = 0.0
    for t, a in enumerate(run["actions"]):
        act = torch.tensor([a], dtype=torch.float32, device="cuda").repeat(n, 1).contiguous()
        obs, rew, te, tr, info = env.step(act)
        ob = obs.cpu().numpy()
        assert np.array_equal(ob, np.tile(ob[:1], (n, 1)))
        assert bool(te[0]) == run["terminated"][t] and bool(tr[0]) == run["truncated"][t], t
        assert bool(te.all()) == bool(te[0]) and bool(tr.all()) == bool(tr[0]) and float(rew.abs().max()) == 0.0
        assert ("final_obs" in info) == (run["final_obs"][t] is not None), t
        if "final_obs" in info:
            fin = info["final_obs"].cpu().numpy()
            assert info["_final_obs"].all()
            worst_fin = max(worst_fin, float(np.abs(fin - np.asarray(run["final_obs"][t])).max()))
        worst_obs = max(worst_obs, float(np.abs(ob[0] - np.asarray(run["obs"][t])).max()))
        worst_v = max(worst_v, abs(float(env.mpc_balancer.commanded_velocity[0]) - run["commanded_velocity"][t]))
    assert worst_obs < 5e-5 and worst_fin < 5e-5, (worst_obs, worst_fin)
    assert worst_v < 2e-2, worst_v
    env.close()


# ---- 4. paths and invariance ----------------------------------------------------------------------------------------

@pytest.mark.parametrize("copy", [True, False])
@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_host_arrays_and_tensors_agree(model, torch, mode, copy):
    n, T = 512, 15
    host, dev = (_env(model, n, mode, max_episode_steps=T, copy=copy) for _ in range(2))
    host.reset(seed=5)
    dev.reset(seed=5)
    rng = np.random.default_rng(0)
    seen = 0
    for k in range(3 * T + 2):
        act = rng.uniform(-0.5, 0.5, (n, 2)).astype(np.float32)
        o, r, te, tr, info = host.step(act)
        do, dr, dte, dtr, dinfo = dev.step_tensors(torch.from_numpy(act).cuda())
        assert isinstance(o, np.ndarray) and te.dtype == np.bool_
        assert np.array_equal(te, dte.cpu().numpy().astype(bool)) and np.array_equal(tr, dtr.cpu().numpy().astype(bool))
        assert np.allclose(o, do.cpu().numpy(), rtol=0, atol=1e-6)
        assert ("final_obs" in info) == ("final_obs" in dinfo), k
        if "final_obs" in info:
            seen += 1
            assert isinstance(info["final_obs"], np.ndarray) and info["final_obs"].shape == (n, 3)
            m = info["_final_obs"]
            assert m.dtype == np.bool_ and np.array_equal(m, dinfo["_final_obs"].cpu().numpy())
            assert np.allclose(info["final_obs"][m], dinfo["final_obs"].cpu().numpy()[m], rtol=0, atol=1e-6)
    assert seen >= (2 if mode == "same_step" else 0)
    host.close()
    dev.close()


@pytest.mark.parametrize("mode", ["next_step", "same_step"])
def test_two_shards_reproduce_one_batch(model, torch, mode):
    n, T = 1024, 25
    whole = _env(model, 2 * n, mode, max_episode_steps=T)
    shards = [_env(model, n, mode, max_episode_steps=T, env_offset=r * n) for r in range(2)]
    for e in [whole] + shards:
        e.reset(seed=9)
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1)
    resets = 0
    for k in range(3 * T):
        act = (torch.rand((2 * n, 2), device="cuda", generator=gen) - 0.5).contiguous()
        o, _, t, r, info = whole.step_tensors(act)
        o, t, r = o.clone(), t.clone(), r.clone()
        fin = info["final_obs"].clone() if "final_obs" in info else None
        for s, sl in zip(shards, (slice(0, n), slice(n, 2 * n))):
            so, _, st, sr, sinfo = s.step_tensors(act[sl].contiguous())
            assert torch.equal(so, o[sl]) and torch.equal(st, t[sl]) and torch.equal(sr, r[sl]), k
            if fin is not None and "final_obs" in sinfo:
                m = sinfo["_final_obs"]
                assert torch.equal(sinfo["final_obs"][m], fin[sl][m]), k
            assert torch.equal(s._xy, whole._xy[sl]), k
        resets += int((t | r).sum())
    assert resets > 0


def test_explicit_reset_cancels_a_pending_next_step_reset(model, torch):
    n, T = 256, 6
    env = _env(model, n, "next_step", max_episode_steps=T)
    env.reset(seed=3)
    act = np.tile(np.array([[0.4, 0.3]], np.float32), (n, 1))
    for k in range(T):
        o, _, te, tr, _ = env.step(act)
    assert tr.all()  # every env has a next-step reset pending
    episode = env.sim.state_dict()["episode"].cpu().clone()
    mask = np.zeros(n, np.uint8)
    mask[::2] = 1
    ro, _ = env.reset(options={"reset_mask": mask})
    assert not ro[::2].any() and np.array_equal(ro[1::2], o[1::2])  # the other envs keep their last observation
    assert not env._xy[::2].any() and env._xy[1::2].abs().min() > 0
    o, _, te, tr, _ = env.step(act)
    ep = env.sim.state_dict()["episode"].cpu()
    # explicitly reset envs: a normal step from their new state; the others: the fused reset step
    assert torch.equal(ep[::2], episode[::2]) and torch.equal(ep[1::2], episode[1::2] + 1)
    assert (np.abs(o[::2, 0]) > 0).all() and not o[1::2].any()
    assert not te.any() and not tr.any()
    env.close()


def test_c_entry_rejects_bad_arguments_without_launching(model, torch):
    from upkie_b200._lib import lib
    from upkie_b200.mpc import BatchedMPCBalancer

    n = 64
    env = _env(model, n, "same_step")
    env.reset(seed=0)
    other = BatchedMPCBalancer(n + 1)
    t = lambda *s: torch.zeros(s, dtype=torch.float32, device="cuda")  # noqa: E731
    action, g6, gf6, obs, fin = t(n, 2), t(n, 6), t(n, 6), t(n, 3), t(n, 3)
    xy = torch.full((n, 2), 7.0, device="cuda")
    env.mpc_balancer.commanded_velocity.fill_(5.0)
    obs.fill_(SENTINEL)

    def args(**kw):
        d = dict(action=action, gyropod_obs=g6, gyropod_final_obs=gf6, xy=xy,
                 commanded_velocity=env.mpc_balancer.commanded_velocity, obs=obs, final_obs=fin)
        d.update(kw)
        a = _abi.UpkieBaseVelocityPost(*[None if d[f] is None else d[f].data_ptr() for f, _ in
                                         _abi.UpkieBaseVelocityPost._fields_[:7]])
        a.dt = kw.get("dt", env.dt)
        a.autoreset_mode = kw.get("mode", 2)
        return C.byref(a)

    L = lib()
    h, m = env.sim._h, env.mpc_balancer._h
    cases = [
        (None, m, args()), (h, None, args()), (h, m, None), (h, other._h, args()),
        (h, m, args(action=None)), (h, m, args(gyropod_obs=None)), (h, m, args(xy=None)),
        (h, m, args(commanded_velocity=None)), (h, m, args(obs=None)),
        (h, m, args(final_obs=None)), (h, m, args(gyropod_final_obs=None)),
        (h, m, args(dt=0.0)), (h, m, args(dt=float("nan"))), (h, m, args(mode=1)), (h, m, args(mode=3)),
    ]
    for k, (hh, mm, aa) in enumerate(cases):
        assert L.upkie_b200_base_velocity_post(hh, mm, aa, None) == -1, k  # UPKIE_B200_EINVAL
        assert L.upkie_b200_last_error(), k
    torch.cuda.synchronize()
    assert (xy == 7.0).all() and (obs == SENTINEL).all() and (env.mpc_balancer.commanded_velocity == 5.0).all()
    assert L.upkie_b200_base_velocity_post(h, m, args(), None) == 0  # the same buffers are accepted
    torch.cuda.synchronize()
    assert (obs != SENTINEL).all()
    other.close()
    env.close()
