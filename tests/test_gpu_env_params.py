# SPDX-License-Identifier: Apache-2.0
"""Per-env parameter table in the step kernels (upkie_b200_set_env_params): a table equal to the config changes no
bit, a heterogeneous batch equals its groups run one by one with their values in the config, the IMU and measurement
noise columns, the vector env, checkpoints and the calls that reject a table."""
import numpy as np
import pytest

from upkie_b200 import UpkieRuntimeError, _abi

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def torch():
    import torch

    assert torch.cuda.is_available()
    return torch


def _headline_config(**kw):
    cfg = _abi.default_sim_config()  # bench.py servos_config
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    for k, v in kw.items():
        setattr(cfg, k, v)
    return cfg


def _sim(model, cfg, n, mode=1, seed=7, env_offset=0, rows=None):
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    if rows is not None:
        s.set_env_params(rows)
    s.set_autoreset(mode, seed, env_offset)
    s.reset(seed=seed, env_offset=env_offset)
    return s


def _config_rows(torch, cfg, n):
    return torch.from_numpy(_abi.config_env_params(cfg)).cuda().expand(n, _abi.EP_DIM).contiguous()


def _servo_actions(torch, model, n, k, seed=3):
    """position targets with velocity targets (gains and friction all act), one set per step"""
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed * 1000 + k)
    a = torch.zeros((n, 6, 6), device="cuda")
    a[:, :, 0] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 0.4
    a[:, :, 1] = (torch.rand((n, 6), device="cuda", generator=gen) * 2 - 1) * 3.0
    a[:, :, 3] = a[:, :, 4] = 1.0
    a[:, :, 5] = torch.tensor(model.tau_max, dtype=torch.float32, device="cuda")
    return a


def _step(torch, model, sim, kind, k):
    n = sim.n
    if kind == "servos":
        out = sim.step_servos(_servo_actions(torch, model, n, k))
    elif kind == "compact":
        out = sim.step_servos_compact_truncated(_servo_actions(torch, model, n, k))
    elif kind == "compact_host":
        out = sim.step_host(_servo_actions(torch, model, n, k).cpu().numpy(), 36, compact=True)[:3]
        return [torch.from_numpy(np.array(x)) for x in out]
    elif kind == "gyropod":
        out = sim.step_gyropod(torch.full((n, 2), 0.3, device="cuda"))
    else:
        out = sim.step_pendulum(torch.full((n, 1), -0.2, device="cuda"))
    return [x.clone() for x in out]


def _assert_same(torch, a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.cpu(), y.cpu())


# ---- identity ---------------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("kind,kw", [
    ("servos", {}), ("compact", {}), ("compact_host", {}), ("gyropod", {}), ("pendulum", {}),
    ("servos", {"spine_mode": 1}), ("servos", {"body_contacts": 1}),
    ("servos", {"torque_control_noise": None}),
])
def test_config_equal_table_is_bit_identical(model, torch, kind, kw):
    kw = dict(kw)
    cfg = _headline_config(**{k: v for k, v in kw.items() if v is not None})
    if "torque_control_noise" in kw:  # noise models on (the extras kernels draw)
        for j in range(6):
            cfg.torque_control_noise[j] = 0.05
            cfg.torque_measurement_noise[j] = 0.02
        cfg.imu_accelerometer_noise = 0.1
    n = 640
    plain = _sim(model, cfg, n)
    table = _sim(model, cfg, n, rows=_config_rows(torch, cfg, n))
    for k in range(12):
        if k == 8:
            table.set_env_params(None)  # and clearing the table again
        _assert_same(torch, _step(torch, model, plain, kind, k), _step(torch, model, table, kind, k))
        _assert_same(torch, [plain.get_state(), plain.spine_obs()], [table.get_state(), table.spine_obs()])


# ---- heterogeneous = grouped homogeneous ------------------------------------------------------------------------------

GROUP = 512


def _group_configs(spine=False):
    out = []
    for g, (kp, kd, fr, cn, mn) in enumerate([(20.0, 1.0, 0.0, 0.0, 0.0), (15.0, 0.6, 0.03, 0.05, 0.02),
                                                (25.0, 1.4, 0.05, 0.0, 0.04), (18.0, 1.2, 0.01, 0.08, 0.0)]):
        cfg = _headline_config(noise_seed=99, spine_mode=1 if spine else 0, fall_pitch=0.25)
        cfg.torque_control_kp, cfg.torque_control_kd = kp, kd
        for j in range(6):
            cfg.joint_friction[j] = fr * (1.0 + 0.2 * j)
            cfg.torque_control_noise[j] = cn
            cfg.torque_measurement_noise[j] = mn
        for k in range(3):
            cfg.imu_accelerometer_bias[k] = 0.01 * g * (k - 1)
            cfg.imu_gyroscope_bias[k] = 0.002 * g
        cfg.imu_accelerometer_noise = 0.05 * g
        cfg.imu_gyroscope_noise = 0.01 * (3 - g)
        out.append(cfg)
    return out


@pytest.mark.parametrize("mode,spine", [(1, False), (2, False), (1, True)])
def test_heterogeneous_table_matches_grouped_handles(model, torch, mode, spine):
    cfgs = _group_configs(spine)
    n = GROUP * len(cfgs)
    rows = torch.cat([_config_rows(torch, c, GROUP) for c in cfgs]).contiguous()
    base = _headline_config(noise_seed=99, spine_mode=1 if spine else 0, fall_pitch=0.25)
    mixed = _sim(model, base, n, mode=mode, rows=rows)
    groups = [_sim(model, c, GROUP, mode=mode, env_offset=GROUP * g) for g, c in enumerate(cfgs)]
    fin_m = torch.zeros((n, 6, 5), device="cuda") if mode == 2 else None
    fin_g = [torch.zeros((GROUP, 6, 5), device="cuda") if mode == 2 else None for _ in groups]

    def check():
        _assert_same(torch, [mixed.get_state(), mixed.spine_obs(), mixed.reset_obs(30)],
                     [torch.cat([s.get_state() for s in groups]), torch.cat([s.spine_obs() for s in groups]),
                      torch.cat([s.reset_obs(30) for s in groups])])

    check()
    resets = 0
    for k in range(40):
        a = _servo_actions(torch, model, n, k)
        out_m = [x.clone() for x in mixed.step_servos(a, final_obs=fin_m)]
        outs = [[x.clone() for x in s.step_servos(a[GROUP * g : GROUP * (g + 1)].contiguous(), final_obs=fin_g[g])]
                for g, s in enumerate(groups)]
        _assert_same(torch, out_m, [torch.cat([o[i] for o in outs]) for i in range(4)])
        resets += int(out_m[2].sum())
        if mode == 2:
            assert torch.equal(fin_m, torch.cat(fin_g))
        check()
    assert resets > 0  # the auto-reset ran inside the window
    # the groups do differ
    st = mixed.get_state()
    assert not torch.equal(st[:GROUP], st[GROUP : 2 * GROUP])


# ---- vector env, checkpoints ------------------------------------------------------------------------------------------

def test_vector_env_with_per_env_gains(model, torch):
    from upkie_b200 import JointProperties
    from upkie_b200.envs import B200VectorEnv

    n = 64
    kp = np.linspace(15.0, 25.0, n)
    props = {"left_knee": JointProperties(friction=np.linspace(0.0, 0.05, n), torque_control_noise=0.02)}
    for tensors in (False, True):
        env = B200VectorEnv(n, "servos", model=model, torque_control_kp=kp, joint_properties=props,
                            autoreset_mode="next_step")
        ref = B200VectorEnv(n, "servos", model=model, autoreset_mode="next_step")
        assert env.sim.get_env_params()[:, _abi.EP_KP].cpu().numpy() == pytest.approx(kp.astype(np.float32))
        env.reset(seed=1)
        ref.reset(seed=1)
        for k in range(5):
            if k == 3:
                # takes effect on the next step: from now on both envs run the same parameters
                env.set_joint_properties({"left_knee": JointProperties()}, torque_control_kp=20.0)
                ref.sim.set_state(env.sim.get_state())
            if tensors:
                a = _servo_actions(torch, model, n, k)
                o1, o2 = env.step_tensors(a)[0], ref.step_tensors(a)[0]
                o1, o2 = o1.cpu().numpy(), o2.cpu().numpy()
            else:
                a = {name: {"position": np.full((n, 1), 0.1), "velocity": np.full((n, 1), 1.0)}
                     for name in _abi.JOINT_NAMES}
                o1, o2 = env.step(a)[0], ref.step(a)[0]
                o1 = np.stack([o1[name]["velocity"] for name in _abi.JOINT_NAMES])
                o2 = np.stack([o2[name]["velocity"] for name in _abi.JOINT_NAMES])
            assert (np.array_equal(o1, o2)) == (k >= 3), k
        env.close()
        ref.close()


def test_checkpoint_round_trip_with_a_table(model, torch):
    cfg = _headline_config(noise_seed=5)
    n = 256
    rows = _config_rows(torch, cfg, n).clone()
    rows[:, _abi.EP_KP] = torch.linspace(15.0, 25.0, n, device="cuda")
    rows[:, _abi.EP_CTRL_NOISE : _abi.EP_CTRL_NOISE + 6] = 0.03
    a = _sim(model, cfg, n, rows=rows)
    for k in range(5):
        _step(torch, model, a, "servos", k)
    sd = a.state_dict()
    b = _sim(model, cfg, n)
    b.load_state_dict(sd)
    assert torch.equal(b.get_env_params(), rows)
    for k in range(5, 10):
        _assert_same(torch, _step(torch, model, a, "servos", k), _step(torch, model, b, "servos", k))
    # a checkpoint written before the table existed loads as "no table"
    old = dict(sd)
    old.pop("env_params")
    b.load_state_dict(old)
    assert torch.equal(b.get_env_params(), _config_rows(torch, cfg, n))
    assert b.state_dict()["env_params"] is None


# ---- rejections -------------------------------------------------------------------------------------------------------

def test_invalid_table_keeps_the_previous_one(model, torch):
    cfg = _headline_config()
    n = 96
    rows = _config_rows(torch, cfg, n).clone()
    rows[:, _abi.EP_KD] = 0.5
    s = _sim(model, cfg, n, rows=rows)
    for col, bad in ((_abi.EP_KP, -1.0), (_abi.EP_FRICTION, float("nan")), (_abi.EP_MEAS_NOISE + 5, -0.1),
                     (_abi.EP_IMU_GYRO_BIAS, float("inf"))):
        r = rows.clone()
        r[n - 1, col] = bad
        with pytest.raises(UpkieRuntimeError, match="error -1"):
            s.set_env_params(r)
        assert torch.equal(s.get_env_params(), rows)


def test_transports_reject_a_table_before_launching(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 64
    cfg = _headline_config()
    s = UpkieSim(n, model=model, config=cfg)
    s.set_env_params(_config_rows(torch, cfg, n))
    s.reset(seed=1)
    obs = torch.zeros((n, 6, 3), device="cuda")
    term = torch.zeros(n, dtype=torch.uint8, device="cuda")
    a = _servo_actions(torch, model, n, 0)
    before = s.launches
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.step_servos_push(a, obs.data_ptr(), term.data_ptr())
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.step_servos_peers(a, [obs.data_ptr()], [term.data_ptr()])
    with pytest.raises(UpkieRuntimeError, match="error -1"):
        s.step_servos_multicast(a, obs.data_ptr(), term.data_ptr())
    assert s.launches == before
