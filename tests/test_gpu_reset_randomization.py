# SPDX-License-Identifier: Apache-2.0
"""Reset randomisation on the device (upkie_b200_set_reset_randomization): the draw law after fused and explicit
resets, equivalence with values written from the host, terminal observations with the old episode's values, GPU-count
invariance, checkpoints, the rejections, and the base-velocity env."""
import numpy as np
import pytest

from upkie_b200 import UpkieRuntimeError, _abi
from test_reset_randomization_cpu import draw_np

pytestmark = pytest.mark.gpu

SEED = 11

# ranges of every column: gains, joint friction, noise, IMU uncertainty, inertia epsilons, floor friction
_RANGES = ([(15.0, 25.0), (0.5, 1.5)] + [(0.0, 0.05)] * 6 + [(0.0, 0.05)] * 6 + [(0.0, 0.05)] * 6
           + [(-0.1, 0.1)] * 3 + [(0.0, 0.05)] + [(-0.01, 0.01)] * 3 + [(0.0, 0.01)] + [(-0.2, 0.2)] * 6 + [(0.6, 1.2)])
ALL = (1 << _abi.RR_DIM) - 1


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _spec(columns=ALL):
    s = _abi.UpkieResetRandomization()
    s.columns = columns
    for k, (lo, hi) in enumerate(_RANGES):
        s.low[k], s.high[k] = lo, hi
    return s


def _config(**kw):
    cfg = _abi.default_sim_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.noise_seed = 5
    cfg.max_episode_steps = 20
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _sim(model, cfg, n, mode, spec=None, env_offset=0):
    """a handle reset once (before the spec: the first values are the config's), then the spec set"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    s.reset(seed=SEED, env_offset=env_offset)
    if spec is not None:
        s.set_reset_randomization(spec)
    return s


def _action(torch, model, kind, n, k, env_offset=0, total=None):
    """random actions of tick k for the envs [env_offset, env_offset + n) of a batch of `total`"""
    total = total or n
    gen = torch.Generator(device="cuda")
    gen.manual_seed(1000 + k)
    if kind == "servos":
        a = torch.zeros((total, 6, 6), device="cuda")
        a[:, :, 0] = (torch.rand((total, 6), device="cuda", generator=gen) * 2 - 1) * 0.6
        a[:, :, 1] = (torch.rand((total, 6), device="cuda", generator=gen) * 2 - 1) * 4.0
        a[:, :, 3] = a[:, :, 4] = 1.0
        a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    else:
        a = (torch.rand((total, 1), device="cuda", generator=gen) * 2 - 1) * 2.0
    return a[env_offset : env_offset + n].contiguous()


def _step(sim, kind, a, **kw):
    out = sim.step_servos(a, **kw) if kind == "servos" else sim.step_pendulum(a, **kw)
    return [x.clone() for x in out]


def _values(sim):
    """[N, RR_DIM] the values in force, in column order"""
    import torch

    fr, eps = sim.get_randomization()
    return torch.cat([sim.get_env_params(), eps, fr[:, None]], dim=1).cpu().numpy()


def _check_law(sim, spec, initial, env_offset=0):
    vals, draws = _values(sim), sim.get_draws().cpu().numpy().astype(np.uint32)
    sel = np.array([(spec.columns >> k) & 1 for k in range(_abi.RR_DIM)], dtype=bool)
    drawn = draws > 0
    expect = draw_np(spec, SEED, env_offset + np.arange(sim.n), draws)
    np.testing.assert_array_equal(vals[drawn][:, sel], expect[drawn][:, sel])
    np.testing.assert_array_equal(vals[:, ~sel], initial[:, ~sel])
    np.testing.assert_array_equal(vals[~drawn], initial[~drawn])
    lo, hi = np.array(_RANGES, dtype=np.float32).T
    assert np.all(vals[drawn][:, sel] >= lo[sel]) and np.all(vals[drawn][:, sel] <= hi[sel])
    return draws


# ---- 1. the draw law ---------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "pendulum"])
@pytest.mark.parametrize("mode", [1, 2])
def test_draw_law_after_fused_resets(model, torch, kind, mode):
    n = 4096
    spec = _spec(ALL & ~(1 << _abi.EP_KD) & ~(1 << (_abi.RR_INERTIA + 3)))  # two columns left alone
    s = _sim(model, _config(), n, mode)
    initial = _values(s)
    s.set_reset_randomization(spec)
    _check_law(s, spec, initial)  # no draw yet
    for k in range(300):
        _step(s, kind, _action(torch, model, kind, n, k))
    draws = _check_law(s, spec, initial)
    assert draws.min() >= 5  # every env reset at least once per time limit


# ---- 2. equivalence with values written from the host ------------------------------------------------------------------


@pytest.mark.parametrize("mode", [1, 2])
@pytest.mark.parametrize("family", ["table", "body"])
def test_drawn_values_act_as_host_written_ones(model, torch, mode, family):
    n, kind = 2048, "servos"
    cfg = _config(body_contacts=1 if family == "body" else 0, joint_limits=2)
    a_sim = _sim(model, cfg, n, mode, _spec())
    k = 20 if mode == 1 else 19  # the tick of the time limit's first resets (and of some falls')
    for t in range(k):
        _step(a_sim, kind, _action(torch, model, kind, n, t))
    before = a_sim.state_dict()
    draws = a_sim.get_draws().clone()
    ref = [_step(a_sim, kind, _action(torch, model, kind, n, k))]
    assert bool((a_sim.get_draws() != draws).any())  # some env reset in this tick
    after = a_sim.state_dict()
    # from here on the spec selects nothing: resets still take the randomisation's path, and change no value
    a_sim.set_reset_randomization(_spec(0))
    if mode == 1:
        # next step: the tick's resets run from its start, with the values drawn for them; the twin gets those values
        # written from the host before the tick and runs the tick itself
        sd = dict(before, env_params=after["env_params"], friction=after["friction"], inertia_eps=after["inertia_eps"])
        ticks = range(k, k + 51)
    else:
        # same step: the draw comes after the tick's physics; the twin starts right after the reset
        sd = dict(after)
        ticks = range(k + 1, k + 51)
        ref = []
    sd["reset_randomization"] = None
    from upkie_b200.sim import UpkieSim

    b_sim = UpkieSim(n, model=model, config=cfg)
    b_sim.load_state_dict(sd)
    outs_b = []
    for t in ticks:
        a = _action(torch, model, kind, n, t)
        if t > k or mode == 2:
            ref.append(_step(a_sim, kind, a))
        outs_b.append(_step(b_sim, kind, a))
    for x, y in zip(ref, outs_b):
        for u, v in zip(x, y):
            assert torch.equal(u, v)
    assert torch.equal(a_sim.get_state(), b_sim.get_state())


# ---- 3. terminal observations keep the old episode's values ------------------------------------------------------------


def test_terminal_observations_use_the_ended_episode_values(model, torch):
    n, kind = 2048, "servos"
    cfg = _config(joint_limits=2)
    a_sim = _sim(model, cfg, n, 2, _spec())
    c_sim = _sim(model, cfg, n, 0)  # the same actions without resets
    c_sim.set_env_params(a_sim.get_env_params())  # the same kernel family, the config's values
    fin = torch.zeros((n, 6, 5), device="cuda")
    seen = torch.zeros(n, dtype=torch.bool, device="cuda")
    checked = 0
    for k in range(40):
        a = _action(torch, model, kind, n, k)
        _, _, term, trunc = _step(a_sim, kind, a, final_obs=fin, final_state=True)
        spine_fin = a_sim.final_spine_obs()
        obs_c = _step(c_sim, kind, a)[0]
        spine_c = c_sim.spine_obs()
        first = (term.bool() | trunc.bool()) & ~seen
        assert torch.equal(fin[first], obs_c[first])
        assert torch.equal(spine_fin[first], spine_c[first])
        checked += int(first.sum())
        seen |= first
    assert checked > n // 2
    # the resets drew new levels, which the envs' observations now use
    assert not torch.equal(a_sim.get_env_params(), c_sim.get_env_params())


# ---- 4. GPU-count invariance -------------------------------------------------------------------------------------------


def test_two_shards_hold_the_tables_of_one_batch(model, torch):
    n, kind = 4096, "pendulum"
    whole = _sim(model, _config(), n, 1, _spec())
    shards = [_sim(model, _config(), n // 2, 1, _spec(), env_offset=o) for o in (0, n // 2)]
    for k in range(100):
        _step(whole, kind, _action(torch, model, kind, n, k))
        for s, o in zip(shards, (0, n // 2)):
            _step(s, kind, _action(torch, model, kind, n // 2, k, o, n))
    np.testing.assert_array_equal(_values(whole), np.concatenate([_values(s) for s in shards]))
    assert torch.equal(whole.get_draws().cpu(), torch.cat([s.get_draws().cpu() for s in shards]))


# ---- 5. explicit resets ------------------------------------------------------------------------------------------------


def test_explicit_resets_through_the_vector_env(torch):
    from upkie_b200.envs import B200VectorEnv

    n = 64
    rr = {"inertia_variation": 0.2, "floor_friction": (0.6, 1.2), "torque_control_kp": (15.0, 25.0),
          "joint_properties": {"left_knee": {"friction": (0.0, 0.05)}},
          "imu_uncertainty": {"gyroscope_bias": ((-0.01, 0.0, -0.02), (0.01, 0.0, 0.02))}}
    env = B200VectorEnv(n, "servos", reset_randomization=rr)
    try:
        env.reset(seed=3)
        first = _values(env.sim)
        assert env.sim.get_draws().cpu().tolist() == [1] * n
        env.reset(seed=3)
        np.testing.assert_array_equal(_values(env.sim), first)
        mask = np.arange(n) % 3 == 0
        env.reset(options={"reset_mask": mask})
        now = _values(env.sim)
        assert env.sim.get_draws().cpu().tolist() == [2 if m else 1 for m in mask]
        np.testing.assert_array_equal(now[~mask], first[~mask])
        assert not np.any(np.all(now[mask] == first[mask], axis=1))
        env.set_reset_randomization(None)
        env.reset(seed=4)
        np.testing.assert_array_equal(_values(env.sim), now)  # off: the values in force stay
    finally:
        env.close()


# ---- 6. checkpoints ----------------------------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n, kind = 1024, "servos"
    cfg = _config()
    a_sim = _sim(model, cfg, n, 1, _spec())
    for k in range(30):
        _step(a_sim, kind, _action(torch, model, kind, n, k))
    b_sim = UpkieSim(n, model=model, config=cfg)
    b_sim.load_state_dict(a_sim.state_dict())
    for k in range(30, 70):
        a = _action(torch, model, kind, n, k)
        for x, y in zip(_step(a_sim, kind, a), _step(b_sim, kind, a)):
            assert torch.equal(x, y)
    np.testing.assert_array_equal(_values(a_sim), _values(b_sim))
    assert torch.equal(a_sim.get_draws(), b_sim.get_draws())
    # a checkpoint without the keys loads as "off, counters 0"
    old = {key: v for key, v in a_sim.state_dict().items() if key not in ("reset_randomization", "draws")}
    b_sim.load_state_dict(old)
    assert b_sim.state_dict()["reset_randomization"] is None
    assert int(b_sim.get_draws().abs().sum()) == 0


# ---- 7. rejections -----------------------------------------------------------------------------------------------------


def test_rejections(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 64
    s0 = UpkieSim(n, model=model, config=_config(joint_limits=0))
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s0.set_reset_randomization(_spec())

    s = _sim(model, _config(max_episode_steps=0), n, 0, _spec(1 << _abi.EP_KP))
    obs = torch.zeros((n, 6, 3), device="cuda")
    term = torch.zeros(n, dtype=torch.uint8, device="cuda")
    a = _action(torch, model, "servos", n, 0)
    before = s.launches
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.step_servos_push(a, obs.data_ptr(), term.data_ptr())
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.step_servos_peers(a, [obs.data_ptr()], [term.data_ptr()])
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.step_servos_multicast(a, obs.data_ptr(), term.data_ptr())
    assert s.launches == before

    for col, lo, hi in ((_abi.EP_KD, -0.1, 1.0), (_abi.EP_FRICTION, 0.1, 0.0), (_abi.EP_MEAS_NOISE, 0.0, np.inf),
                        (_abi.EP_IMU_ACC_BIAS, np.nan, 0.0), (_abi.RR_INERTIA, -1.0, 0.0), (_abi.RR_FRICTION, -0.1, 1.0)):
        bad = _spec(ALL)
        bad.low[col], bad.high[col] = lo, hi
        with pytest.raises(UpkieRuntimeError, match="error -1"):
            s.set_reset_randomization(bad)
    # the previous spec (kp only) is still the one in force
    s.reset(seed=SEED)
    vals = _values(s)
    draws = s.get_draws().cpu().numpy().astype(np.uint32)
    np.testing.assert_array_equal(vals[:, _abi.EP_KP], draw_np(_spec(), SEED, np.arange(n), draws)[:, _abi.EP_KP])
    np.testing.assert_array_equal(vals[:, _abi.EP_KD], np.float32(1.0))

    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.set_env_params(None)
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.set_randomization(None, None)
    s.set_reset_randomization(None)
    s.set_env_params(None)  # accepted once the spec is off


# ---- 8. base velocity --------------------------------------------------------------------------------------------------


def test_base_velocity_env_draws_at_its_resets(torch):
    from upkie_b200.envs import B200VectorEnv

    n = 256
    rr = {"torque_control_kp": (15.0, 25.0), "floor_friction": (0.6, 1.2), "inertia_variation": 0.1}
    env = B200VectorEnv(n, "base_velocity", autoreset_mode="next_step", max_episode_steps=15, reset_randomization=rr)
    try:
        env.reset(seed=SEED)
        rng = np.random.default_rng(0)
        for _ in range(60):
            env.step(rng.uniform(-1.0, 1.0, (n, 2)).astype(np.float32))
        spec = env.sim._reset_randomization
        vals = _values(env.sim)
        draws = env.sim.get_draws().cpu().numpy().astype(np.uint32)
        assert draws.min() >= 4
        sel = np.array([(spec.columns >> k) & 1 for k in range(_abi.RR_DIM)], dtype=bool)
        np.testing.assert_array_equal(vals[:, sel], draw_np(spec, SEED, np.arange(n), draws)[:, sel])
    finally:
        env.close()
