# SPDX-License-Identifier: Apache-2.0
"""info["final_info"] of same-step auto-resets on the GPU: the terminal spine observation the step kernel stashes
(UpkieStepOutputs.final_state, upkie_b200_final_spine_obs) against a twin without auto-reset, in every step kind;
the vector env's keys and masks on the host and device paths; base_velocity envs; a stash that does not disturb the
step; and the calls that refuse to return stale rows."""
import ctypes as C

import numpy as np
import pytest

from upkie_b200 import _abi

pytestmark = pytest.mark.gpu

SENTINEL = -12345.0
# columns differentiated from velocities over one tick: their round-off is that of a velocity divided by the tick
ACC_COLUMNS = list(range(_abi.SP_IMU_LINACC, _abi.SP_IMU_LINACC + 3)) + list(range(_abi.SP_IMU_RAWACC, _abi.SP_IMU_RAWACC + 3))


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _sim(n, model, cfg, mode, seed=7):
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, seed, 0)
    s.reset(seed=seed)
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
    a = torch.zeros((n, 6, 6), device="cuda")
    a[:, :, 0] = float("nan")
    a[:, :, 5] = tau
    a[:, :, 2] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * tau
    return a


def _env_params(torch, cfg, n, seed):
    """A per-env table with torque measurement noise and IMU uncertainty that differ from env to env."""
    rng = np.random.default_rng(seed)
    rows = np.tile(_abi.config_env_params(cfg).astype(np.float32), (n, 1))
    rows[:, _abi.EP_MEAS_NOISE:_abi.EP_MEAS_NOISE + 6] = rng.uniform(0.0, 0.5, (n, 6))
    rows[:, _abi.EP_IMU_ACC_BIAS:_abi.EP_IMU_ACC_BIAS + 3] = rng.uniform(-0.2, 0.2, (n, 3))
    rows[:, _abi.EP_IMU_GYRO_BIAS:_abi.EP_IMU_GYRO_BIAS + 3] = rng.uniform(-0.05, 0.05, (n, 3))
    rows[:, _abi.EP_IMU_ACC_NOISE] = rng.uniform(0.0, 0.3, n)
    rows[:, _abi.EP_IMU_GYRO_NOISE] = rng.uniform(0.0, 0.02, n)
    return torch.from_numpy(rows).cuda().contiguous()


def _case(torch, model, kind):
    """(config, n, step(sim, k, final_state) -> (terminated, truncated) on the host, per-handle setup)."""
    n = 4096
    cfg = _headline_config(40)
    cfg.rand_pitch = 0.6  # some robots fall before their first time-out
    setup = None
    if kind in ("servos", "compact", "host_compact", "spine", "table", "body"):
        if kind == "spine":
            cfg.spine_mode = 1
        if kind == "body":
            cfg.body_contacts = 1
        if kind == "table":
            table = _env_params(torch, cfg, n, 3)
            setup = lambda s: s.set_env_params(table)  # noqa: E731
        acts = [_torque_actions(torch, model, n, 11 + j) for j in range(4)]
        if kind == "compact":
            def step(s, k, fs):
                _, t, r = s.step_servos_compact_truncated(acts[k % 4], final_state=fs)
                return t.cpu().bool(), r.cpu().bool()
        elif kind == "host_compact":
            host = [x.cpu().numpy() for x in acts]

            def step(s, k, fs):
                _, t, r, _ = s.step_host(host[k % 4], 36, compact=True, final_state=fs)
                return torch.from_numpy(t.copy()).bool(), torch.from_numpy(r.copy()).bool()
        else:
            def step(s, k, fs):
                _, _, t, r = s.step_servos(acts[k % 4], final_state=fs)
                return t.cpu().bool(), r.cpu().bool()
    else:
        # full ground velocity, one direction per env: the robots that do not fall within the limit time out
        cfg.max_episode_steps = 80
        dim = 2 if kind == "gyropod" else 1
        gen = torch.Generator(device="cuda")
        gen.manual_seed(5)
        act = (3.0 * torch.where(torch.rand((n, dim), device="cuda", generator=gen) < 0.5, -1.0, 1.0)).contiguous()
        fn = "step_gyropod" if kind == "gyropod" else "step_pendulum"

        def step(s, k, fs):
            _, _, t, r = getattr(s, fn)(act, final_state=fs)
            return t.cpu().bool(), r.cpu().bool()
    return cfg, n, step, setup


def _close(torch, x, y):
    """fp32 round-off of the gyropod / pendulum kernels of two auto-reset modes, which are compiled apart."""
    tol = 1e-5 + 1e-4 * y.abs()
    tol[:, ACC_COLUMNS] += 2e-3
    return bool(((x - y).abs() <= tol).all())


# ---- 1. the twin without auto-reset ------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind", ["servos", "compact", "host_compact", "gyropod", "pendulum", "spine", "table", "body"])
def test_final_spine_obs_equals_the_twin_without_autoreset(model, torch, kind):
    """On its first reset, an env's terminal row is the spine observation its twin (auto-reset disabled, same actions)
    returns after the same step: bit for bit for the servo kinds, to round-off for gyropod and pendulum. The rows of
    the envs that did not reset keep the caller's sentinel."""
    cfg, n, step, setup = _case(torch, model, kind)
    exact = kind not in ("gyropod", "pendulum")
    a = _sim(n, model, cfg, 2)
    b = _sim(n, model, cfg, 0)
    if setup:
        setup(a)
        setup(b)
    out = torch.empty((n, _abi.SPINE_DIM), dtype=torch.float32, device="cuda")
    first = torch.zeros(n, dtype=torch.bool)  # env has reset once: from there on it differs from the twin
    reasons = set()
    for k in range(2 * cfg.max_episode_steps + 20):
        ta, ra = step(a, k, True)
        tb, _ = step(b, k, False)
        out.fill_(SENTINEL)
        fa = a.final_spine_obs(out).cpu()
        sb = b.spine_obs().cpu()
        reset = ta | ra
        fresh = reset & ~first
        assert torch.equal(ta[~first], tb[~first]), k
        assert (fa[~reset] == SENTINEL).all(), (kind, k)
        if exact:
            assert torch.equal(fa[fresh], sb[fresh]), (kind, k)
        else:
            assert _close(torch, fa[fresh], sb[fresh]), (kind, k)
        if fresh.any():
            reasons |= {"fall"} if (ta & fresh).any() else set()
            reasons |= {"time-out"} if (ra & ~ta & fresh).any() else set()
        first |= reset
    assert first.all() and reasons == {"fall", "time-out"}, (int(first.sum()), reasons)


# ---- 2. vector env: keys, masks, host and device paths --------------------------------------------------------------

def _pendulum_policy(o):
    """README policy: keeps the pendulum envs up."""
    n = o.shape[0]
    return (10.0 * o[:, 0] + 1.0 * o[:, 1] + 0.0 * o[:, 2] + 0.1 * o[:, 3]).reshape(n, 1).astype(np.float32)


@pytest.mark.parametrize("copy", [True, False])
@pytest.mark.parametrize("env_type", ["servos", "pendulum"])
def test_vector_env_final_info_host_and_tensors(model, torch, env_type, copy):
    """Host arrays and device tensors give the same keys and masks on the same steps (the actions keep every robot up,
    so every reset is a time-out and both paths reset the same envs); the terminal rows agree to the round-off between
    the shared-memory-tile kernels of the host path and the device-buffer ones; the lazy rows refuse to be read once
    the env has stepped again."""
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.exceptions import UpkieRuntimeError

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
        _, _, dte, dtr, dinfo = dev.step_tensors(torch.from_numpy(act).cuda())
        for i in (info, dinfo):
            assert ("final_info" in i) == ("_final_info" in i) == ("final_obs" in i) == (k % T == 0), k
        if "final_info" not in info:
            continue
        seen += 1
        mask = info["_final_obs"]
        for i in (info, dinfo):
            fi = i["final_info"]
            assert set(fi) == {"spine_observation", "_spine_observation"}
        assert isinstance(info["_final_info"], np.ndarray) and info["_final_info"].dtype == np.bool_
        assert dinfo["_final_info"].is_cuda and dinfo["_final_info"].dtype == torch.bool
        for m in (info["_final_info"], info["final_info"]["_spine_observation"]):
            assert np.array_equal(m, mask)
        for m in (dinfo["_final_info"], dinfo["final_info"]["_spine_observation"], dinfo["_final_obs"]):
            assert np.array_equal(m.cpu().numpy(), mask)
        hf, df = info["final_info"]["spine_observation"], dinfo["final_info"]["spine_observation"]
        assert len(hf) == n and hf.tensor.is_cuda and tuple(hf.tensor.shape) == (n, _abi.SPINE_DIM)
        i0 = int(np.flatnonzero(mask)[0])
        ref = info["spine_observation"][i0]
        for d in (hf[i0], df[i0]):
            assert d.keys() == ref.keys()
            assert all(d[key].keys() == ref[key].keys() for key in ref)
        # the terminal rows are not the reset's rows
        assert not np.array_equal(hf.array[mask], info["spine_observation"].array[mask])
        diff = np.abs(hf.array[mask] - df.array[mask])
        assert np.median(diff) < 1e-4, np.median(diff)
        break
    assert seen >= 1
    # an object not read before the next step raises
    for k in range(3 * T):
        o, _, te, tr, info = host.step(act if env_type == "servos" else _pendulum_policy(o))
        if "final_info" in info:
            lazy = info["final_info"]["spine_observation"]
            host.step(act if env_type == "servos" else _pendulum_policy(o))
            with pytest.raises(UpkieRuntimeError):
                lazy.array
            break
    else:
        raise AssertionError("no reset")
    host.close()
    dev.close()


@pytest.mark.parametrize("path", ["host", "tensors"])
def test_fallen_envs_report_their_terminal_pitch(model, torch, path):
    """Pendulum envs driven at full ground velocity fall: the terminal rows of the fallen envs show a pitch beyond
    fall_pitch (the same-step reset's own rows show the new upright episode)."""
    from upkie_b200.envs import B200VectorEnv

    n = 1024
    env = B200VectorEnv(n, "pendulum", model=model, autoreset_mode="same_step")
    env.reset(seed=3)
    sign = np.where(np.random.default_rng(0).random((n, 1)) < 0.5, -1.0, 1.0).astype(np.float32)
    act = 3.0 * sign
    falls = 0
    for k in range(300):
        if path == "host":
            _, _, te, tr, info = env.step(act)
        else:
            _, _, te, tr, info = env.step_tensors(torch.from_numpy(act).cuda())
            te, tr = te.cpu().numpy().astype(bool), tr.cpu().numpy().astype(bool)
        assert ("final_info" in info) == bool((te | tr).any())
        if "final_info" not in info:
            continue
        rows = info["final_info"]["spine_observation"].array
        pitch = np.abs(rows[te, _abi.SP_PITCH])
        assert (pitch > 1.0 - 1e-4).all(), pitch.min()  # fall_pitch = 1 rad
        assert (np.abs(info["spine_observation"].array[te, _abi.SP_PITCH]) < 0.5).all()
        falls += int(te.sum())
    assert falls > 0
    env.close()


# ---- 3. base_velocity same-step -----------------------------------------------------------------------------------------

def test_base_velocity_final_info_equals_the_masked_reset_twin(model, torch):
    """The terminal spine rows of UpkieBaseVelocity envs are those of the gyropod step that ended the episode: the
    twin without auto-reset, reset by mask like a Gymnasium loop, returns them in info["spine_observation"] before its
    reset (tolerance of tests/test_gpu_base_velocity_autoreset.py, as the gyropod kernels of two modes differ)."""
    from upkie_b200 import ExternalForce
    from upkie_b200.envs import B200VectorEnv

    n, T = 4096, 80
    a = B200VectorEnv(n, "base_velocity", model=model, autoreset_mode="same_step", max_episode_steps=T)
    b = B200VectorEnv(n, "base_velocity", model=model, autoreset_mode="disabled", max_episode_steps=T)
    rng = np.random.default_rng(3)
    push = np.zeros((n, 3))
    push[::2, 0] = rng.uniform(20.0, 200.0, n)[::2]  # half the envs: forward pushes of many sizes, some fall
    for e in (a, b):
        e.reset(seed=2)
        e.set_external_forces({"torso": ExternalForce(push)})
    act = torch.tensor([[0.3, 0.5]], device="cuda").repeat(n, 1).contiguous()
    first = torch.zeros(n, dtype=torch.bool)
    reasons = set()
    for k in range(2 * T + 20):
        _, _, ta, ra, info = a.step_tensors(act)
        _, _, tb, rb, binfo = b.step_tensors(act)
        ta, ra, tb, rb = ta.cpu().bool(), ra.cpu().bool(), tb.cpu().bool(), rb.cpu().bool()
        ended = ta | ra
        assert torch.equal(ta[~first], tb[~first]) and torch.equal(ra[~first], rb[~first]), k
        assert ("final_info" in info) == bool(ended.any()), k
        if ended.any():
            assert torch.equal(info["_final_info"].cpu(), ended)
            fresh = ended & ~first
            rows = info["final_info"]["spine_observation"].tensor.cpu()
            twin = binfo["spine_observation"].tensor.cpu()
            assert _close(torch, rows[fresh], twin[fresh]), k
            reasons |= {"fall"} if (ta & fresh).any() else set()
            reasons |= {"time-out"} if (ra & ~ta & fresh).any() else set()
        first |= ended
        done = (tb | rb).numpy()
        if done.any():
            b.reset(options={"reset_mask": done})
    assert first.all() and reasons == {"fall", "time-out"}, (int(first.sum()), reasons)
    a.close()
    b.close()


# ---- 4. the stash does not disturb the step; stale rows are refused -------------------------------------------------------

def test_stash_does_not_disturb_the_step(model, torch):
    """Two same-step handles, same seed, one with the stash and one without: observations, flags, final-observation
    rows and states stay bit-identical over 200 ticks with resets."""
    n = 4096
    a, b = _sim(n, model, _headline_config(40), 2), _sim(n, model, _headline_config(40), 2)
    acts = [_torque_actions(torch, model, n, 21 + j) for j in range(4)]
    fa = torch.zeros((n, 6, 5), device="cuda")
    fb = torch.zeros((n, 6, 5), device="cuda")
    resets = 0
    for k in range(200):
        oa, _, ta, ra = [x.clone() for x in a.step_servos(acts[k % 4], final_obs=fa, final_state=True)]
        ob, _, tb, rb = b.step_servos(acts[k % 4], final_obs=fb)
        assert torch.equal(oa, ob) and torch.equal(ta, tb) and torch.equal(ra, rb), k
        assert torch.equal(fa, fb), k
        if k % 20 == 19:
            assert torch.equal(a.get_state(), b.get_state()), k
        resets += int((ta | ra).sum())
    assert resets > n  # every env reset at least once on average


def test_no_stash_without_the_flag_and_stale_rows_are_refused(model, torch):
    from upkie_b200.exceptions import UpkieRuntimeError

    n = 65536
    cfg = _headline_config(40)
    s = _sim(n, model, cfg, 2)
    act = _torque_actions(torch, model, n, 5)
    s.step_servos(act)
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    for _ in range(3):
        s.step_servos(act)
    torch.cuda.synchronize()
    assert abs(torch.cuda.mem_get_info()[0] - free0) < (2 << 20)  # no stash: (1 + 50) x 4 B x 65 536 = 13 MB
    with pytest.raises(UpkieRuntimeError, match="final_state"):
        s.final_spine_obs()  # a step without the flag
    s.step_servos(act, final_state=True)
    torch.cuda.synchronize()
    assert free0 - torch.cuda.mem_get_info()[0] >= 12 << 20  # the stash, allocated on the first request
    s.final_spine_obs()
    s.final_spine_obs()  # reading again is fine: nothing moved
    s.reset(seed=1)
    with pytest.raises(UpkieRuntimeError, match="final_state"):
        s.final_spine_obs()  # an explicit reset
    s.step_servos(act, final_state=True)
    s.set_state(s.get_state())
    with pytest.raises(UpkieRuntimeError, match="final_state"):
        s.final_spine_obs()  # set_state
    s.step_servos(act, final_state=True)
    s.load_state_dict(s.state_dict())
    with pytest.raises(UpkieRuntimeError, match="final_state"):
        s.final_spine_obs()  # load_state_dict
    s.close()
    # the flag is ignored outside same-step mode
    s = _sim(256, model, cfg, 1)
    s.step_servos(_torque_actions(torch, model, 256, 5), final_state=True)
    with pytest.raises(UpkieRuntimeError, match="final_state"):
        s.final_spine_obs()
    s.close()


def test_in_kernel_transports_carry_no_stash(model, torch):
    """The in-kernel rollout transports take no UpkieStepOutputs: a step through one of them (here the deferred push
    with nothing to send, a single-GPU call) leaves nothing to read, and the library refuses the rows."""
    from upkie_b200._lib import lib

    n = 256
    s = _sim(n, model, _headline_config(0), 2)
    act = _torque_actions(torch, model, n, 5)
    obs = torch.zeros((n, 6, 3), device="cuda")
    term = torch.zeros(n, dtype=torch.uint8, device="cuda")
    out = torch.zeros((n, _abi.SPINE_DIM), device="cuda")
    p = lambda t: C.c_void_p(t.data_ptr())  # noqa: E731
    s.step_servos(act, final_state=True)
    assert lib().upkie_b200_final_spine_obs(s._h, p(out), None) == 0
    launches = s.launches
    assert lib().upkie_b200_step_servos_push(s._h, p(act), p(obs), p(term), None, None) == 0
    assert s.launches == launches + 1
    assert lib().upkie_b200_final_spine_obs(s._h, p(out), None) == -1
    assert b"final_state" in lib().upkie_b200_last_error()
    assert lib().upkie_b200_final_spine_obs(None, p(out), None) == -1
    assert lib().upkie_b200_final_spine_obs(s._h, None, None) == -1
    torch.cuda.synchronize()
    s.close()
