# SPDX-License-Identifier: Apache-2.0
"""IMU mounting misalignment on the device (upkie_b200_set_imu_misalignment): the physics does not depend on it; every
orientation-derived output is that of the twin's state read through the env's misalignment (an fp64 restatement that
tilts the IMU frame); zero ranges change nothing; the draws follow the NumPy law over fused, explicit, masked, sharded
and chunked host-buffer resets; same-step terminal observations keep the terminal episode's misalignment; the
composition with the observation delay, the history, servo dropouts, IMU bias, the action delay and pushes; the
BaseVelocity MPC input; checkpoints; the rejections."""
import numpy as np
import pytest
import torch as torch_mod
from scipy.spatial.transform import Rotation

from upkie_b200 import UpkieException, UpkieRuntimeError, _abi
from test_imu_misalignment_cpu import RBI, angles_np, quat_np

pytestmark = pytest.mark.gpu

SEED = 0x7117
NEXT_STEP, SAME_STEP = 1, 2
# base_orientation (pitch, rotation) and imu (angular velocity) columns, and two that the misalignment leaves alone
ORIENT_HISTORY = [_abi.SP_PITCH, *range(_abi.SP_ROT, _abi.SP_ROT + 9), *range(_abi.SP_IMU_ANGVEL, _abi.SP_IMU_ANGVEL + 3),
                  _abi.SP_SERVO, _abi.SP_ODOM_POS]
TILT = ((-0.05, 0.05), (-0.1, 0.1), (-0.2, 0.2))
FINAL_SHAPE = {"servos": (6, 5), "gyropod": (6,), "pendulum": (4,)}
UNTOUCHED = [*range(_abi.SP_BASE_LINVEL, _abi.SP_BASE_LINVEL + 3), *range(_abi.SP_IMU_RAWACC + 3, _abi.SPINE_DIM)]


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


def _sim(model, cfg, n, mode, tilt=None, history=ORIENT_HISTORY, sense=None, env_offset=0, drop=(0.0, 0.0)):
    """a handle reset once; a zero-probability servo-dropout spec runs it in FAM_SENSE, so that a twin without the
    misalignment runs the same kernels"""
    from upkie_b200.sim import UpkieSim

    s = UpkieSim(n, model=model, config=cfg)
    s.set_autoreset(mode, SEED, env_offset)
    if history:
        s.set_history(history, 3)
    if sense is not None:
        s.set_observation_delay(*sense)
    if drop is not None:
        s.set_servo_dropout(*drop)
    if tilt is not None:
        s.set_imu_misalignment(*tilt)
    s.reset(seed=SEED, env_offset=env_offset)
    torch_mod.cuda.synchronize()
    return s


def _action(torch, model, kind, n, k):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(9000 + k)
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


def _quat(sim):
    return sim.get_imu_misalignment_state()[1].cpu().numpy().astype(np.float64)


def _counters(sim):
    sd = sim.state_dict()
    return [sd[k].cpu().numpy() for k in ("tick", "episode")]


def tilt_spine(spine, e, bias=(np.zeros(3), np.zeros(3))):
    """fp64: the spine rows a misaligned IMU reports, from the rows `spine` [n, SPINE_DIM] of the same states observed
    by a nominal one and the misalignments e [n, 4]. The nominal IMU frame is Rbi-rotated from the base; the tilted
    one reads every vector through M = Rbi E^T Rbi^T, the observers derive the base rotation R E. `bias` (acc, gyro):
    the IMU bias both rows carry, added in the true IMU frame."""
    s = np.asarray(spine, dtype=np.float64)
    n = len(s)
    E = Rotation.from_quat(np.asarray(e, dtype=np.float64), scalar_first=True).as_matrix()
    R = s[:, _abi.SP_ROT:_abi.SP_ROT + 9].reshape(n, 3, 3)
    RE = R @ E
    M = RBI @ np.transpose(E, (0, 2, 1)) @ RBI.T
    out = s.copy()
    out[:, _abi.SP_ROT:_abi.SP_ROT + 9] = RE.reshape(n, 9)
    out[:, _abi.SP_PITCH] = -np.arcsin(np.clip(RE[:, 2, 0], -1.0, 1.0))
    out[:, _abi.SP_BASE_ANGVEL:_abi.SP_BASE_ANGVEL + 3] = np.einsum(
        "nji,nj->ni", E, s[:, _abi.SP_BASE_ANGVEL:_abi.SP_BASE_ANGVEL + 3])
    for col, b in ((_abi.SP_IMU_ANGVEL, bias[1]), (_abi.SP_IMU_LINACC, bias[0]), (_abi.SP_IMU_RAWACC, bias[0])):
        out[:, col:col + 3] = np.einsum("nij,nj->ni", M, s[:, col:col + 3] - b) + b
    riw = RE @ RBI.T
    out[:, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4] = Rotation.from_matrix(
        np.diag([1.0, -1.0, -1.0]) @ riw).as_quat(scalar_first=True)
    return out


def check_spine(got, ref, label=""):
    """orientation columns of spine rows against tilt_spine: the rotation, sin(pitch) (the pitch itself is steep near
    +-pi/2, where a fallen robot lies), the rates and accelerations, the IMU quaternion up to its sign"""
    np.testing.assert_allclose(got[:, _abi.SP_ROT:_abi.SP_ROT + 9], ref[:, _abi.SP_ROT:_abi.SP_ROT + 9], atol=3e-5,
                               err_msg=label)
    np.testing.assert_allclose(np.sin(got[:, _abi.SP_PITCH].astype(np.float64)), np.sin(ref[:, _abi.SP_PITCH]),
                               atol=3e-5, err_msg=label)
    for col in (_abi.SP_BASE_ANGVEL, _abi.SP_IMU_ANGVEL, _abi.SP_IMU_LINACC, _abi.SP_IMU_RAWACC):
        np.testing.assert_allclose(got[:, col:col + 3], ref[:, col:col + 3], atol=2e-4, rtol=2e-4, err_msg=label)
    q = got[:, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4].astype(np.float64)
    r = ref[:, _abi.SP_IMU_QUAT:_abi.SP_IMU_QUAT + 4]
    sign = np.where(np.sum(q * r, axis=1) < 0, -1.0, 1.0)[:, None]
    np.testing.assert_allclose(q * sign, r, atol=3e-5, err_msg=label)


def check_gyropod(got, twin_spine, e, kind, label=""):
    """gyropod / pendulum rows: the pitch and its rate of the tilted base, the rest as the twin's spine rows give it"""
    ref = tilt_spine(twin_spine, e)
    pitch, rate = (got[:, 1], got[:, 4]) if kind == "gyropod" else (got[:, 0], got[:, 2])
    np.testing.assert_allclose(np.sin(pitch.astype(np.float64)), np.sin(ref[:, _abi.SP_PITCH]), atol=3e-5,
                               err_msg=label)
    np.testing.assert_allclose(rate, ref[:, _abi.SP_BASE_ANGVEL + 1], atol=2e-4, rtol=2e-4, err_msg=label)


def check_history(got, twin, e, label=""):
    """history rows [n, K, C] of ORIENT_HISTORY against the twin's through e"""
    c_rot = ORIENT_HISTORY.index(_abi.SP_ROT)
    c_gyro = ORIENT_HISTORY.index(_abi.SP_IMU_ANGVEL)
    for k in range(got.shape[1]):
        s = np.zeros((len(got), _abi.SPINE_DIM))
        for c, col in enumerate(ORIENT_HISTORY):
            s[:, col] = twin[:, k, c]
        s[:, _abi.SP_IMU_QUAT] = 1.0
        ref = tilt_spine(s, e)
        np.testing.assert_allclose(got[:, k, c_rot:c_rot + 9], ref[:, _abi.SP_ROT:_abi.SP_ROT + 9], atol=3e-5,
                                   err_msg=label)
        np.testing.assert_allclose(np.sin(got[:, k, 0].astype(np.float64)), np.sin(ref[:, _abi.SP_PITCH]), atol=3e-5,
                                   err_msg=label)
        np.testing.assert_allclose(got[:, k, c_gyro:c_gyro + 3], ref[:, _abi.SP_IMU_ANGVEL:_abi.SP_IMU_ANGVEL + 3],
                                   atol=2e-4, rtol=2e-4, err_msg=label)
        # the servo and odometry columns are the twin's
        assert _bits(got[:, k, -2:]) == _bits(twin[:, k, -2:]), label


# ---- 1. the physics does not depend on the misalignment -------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_physics_is_unaffected(model, torch, kind, mode):
    n, T = 256, 300
    cfg = _config()
    sim = _sim(model, cfg, n, mode, tilt=TILT)
    twin = _sim(model, cfg, n, mode)
    resets = 0
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        x = _step(sim, kind, a, same_step=mode == SAME_STEP)
        y = _step(twin, kind, a, same_step=mode == SAME_STEP)
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
        if kind == "servos":
            assert _bits(x[0]) == _bits(y[0]), k  # servo rows carry no orientation
        assert _bits(x[5][:, UNTOUCHED]) == _bits(y[5][:, UNTOUCHED]), k  # servos, odometry, contact, linear velocity
        resets += int((x[1] | x[2]).sum())
    for u, v in zip(_counters(sim), _counters(twin)):
        assert _bits(u) == _bits(v)
    assert resets > 0
    assert not np.array_equal(x[5][:, _abi.SP_PITCH], y[5][:, _abi.SP_PITCH])


# ---- 2, 5. orientation outputs, episode boundaries --------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_orientation_outputs_and_episode_boundaries(model, torch, kind):
    n, T = 512, 60
    cfg = _config(max_episode_steps=9)
    sim = _sim(model, cfg, n, SAME_STEP, tilt=TILT)
    twin = _sim(model, cfg, n, SAME_STEP)
    check_spine(sim.spine_obs().cpu().numpy(), tilt_spine(twin.spine_obs().cpu().numpy(), _quat(sim)), "reset")
    resets = 0
    for k in range(T):
        e_old = _quat(sim)
        a = _action(torch, model, kind, n, k)
        x = _step(sim, kind, a, same_step=True)
        y = _step(twin, kind, a, same_step=True)
        e = _quat(sim)
        done = (x[1] | x[2]).astype(bool)
        resets += int(done.sum())
        assert not np.array_equal(e[done], e_old[done]) or not done.any()
        assert np.array_equal(e[~done], e_old[~done])
        # the observation after the step: the new episode's e_i where a reset happened
        check_spine(x[5], tilt_spine(y[5], e), str(k))
        check_history(x[6], y[6], e, str(k))
        if kind != "servos":
            check_gyropod(x[0], y[5], e, kind, str(k))
        if done.any():
            # the terminal step: the terminal episode's e_i
            check_spine(x[4][done], tilt_spine(y[4][done], e_old[done]), f"final {k}")
            if kind != "servos":
                check_gyropod(x[3][done], y[4][done], e_old[done], kind, f"final {k}")
            else:
                assert _bits(x[3][done]) == _bits(y[3][done])
    assert resets > 0


def test_pure_pitch_offset_adds_to_the_pitch(model, torch):
    n, T = 1024, 30
    cfg = _config(max_episode_steps=0, rand_pitch=0.1)
    spec = ((0.0, 0.0), (-0.08, 0.08), (0.0, 0.0))
    sim = _sim(model, cfg, n, 0, tilt=spec, history=None)
    twin = _sim(model, cfg, n, 0, history=None)
    delta = angles_np(_abi.UpkieImuMisalignment(0, 0, -0.08, 0.08, 0, 0), SEED, np.arange(n), 1)[:, 1]
    for k in range(T):
        a = torch.zeros((n, 2), device="cuda")
        x = sim.step_gyropod(a)[0].cpu().numpy()
        y = twin.step_gyropod(a)[0].cpu().numpy()
    spine = twin.spine_obs().cpu().numpy()
    R = spine[:, _abi.SP_ROT:_abi.SP_ROT + 9].reshape(n, 3, 3)
    roll = np.arctan2(R[:, 2, 1], R[:, 2, 2])
    wheels = np.abs(roll) < 0.02  # on both wheels
    assert wheels.sum() > n // 2
    np.testing.assert_allclose(x[wheels, 1] - y[wheels, 1], delta[wheels], atol=2e-3)
    np.testing.assert_allclose(sim.spine_obs().cpu().numpy()[wheels, _abi.SP_PITCH] - spine[wheels, _abi.SP_PITCH],
                               delta[wheels], atol=2e-3)


# ---- 3. zero ranges: every output of the twin, bit for bit -------------------------------------------------------------


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
@pytest.mark.parametrize("kind", ["servos", "gyropod", "pendulum"])
def test_zero_ranges_match_the_twin(model, torch, kind, mode):
    n, T = 512, 60
    cfg = _config()
    sim = _sim(model, cfg, n, mode, tilt=((0.0, 0.0), (0.0, 0.0), (0.0, 0.0)))
    twin = _sim(model, cfg, n, mode)
    for k in range(T):
        a = _action(torch, model, kind, n, k)
        for x, y in zip(_step(sim, kind, a, same_step=mode == SAME_STEP), _step(twin, kind, a, same_step=mode == SAME_STEP)):
            assert (x is None) == (y is None)
            if x is not None:
                assert _bits(x) == _bits(y), k
        assert _bits(_state(sim)) == _bits(_state(twin)), k
    for kind_dim in (4, 6, 30):
        assert _bits(sim.reset_obs(kind_dim).cpu().numpy()) == _bits(twin.reset_obs(kind_dim).cpu().numpy())
    np.testing.assert_array_equal(_quat(sim), np.tile([1.0, 0.0, 0.0, 0.0], (n, 1)))


# ---- 4. the draws -------------------------------------------------------------------------------------------------------


def _law(spec_tuple, g, count, seed=SEED):
    spec = _abi.UpkieImuMisalignment(*(v for r in spec_tuple for v in r))
    out = np.tile([1.0, 0.0, 0.0, 0.0], (len(g), 1))
    for k in np.unique(count):
        if k == 0:
            continue
        m = count == k
        out[m] = quat_np(angles_np(spec, seed, g[m], k))
    return out


@pytest.mark.parametrize("mode", [NEXT_STEP, SAME_STEP])
def test_draws_follow_the_law(model, torch, mode):
    n, T, off = 512, 80, 1000
    cfg = _config(max_episode_steps=11)
    sim = _sim(model, cfg, n, mode, tilt=TILT, env_offset=off, history=None)
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
    count, quat = sim.get_imu_misalignment_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    assert expect.max() > 2
    np.testing.assert_allclose(quat.cpu().numpy(), _law(TILT, g, expect), atol=2e-6)
    # explicit resets: masked, then with host rows
    mask = torch.zeros(n, dtype=torch.uint8, device="cuda")
    mask[::3] = 1
    sim.reset(mask=mask, seed=5, env_offset=off)
    m = mask.cpu().numpy().astype(bool)
    expect[m] += 1
    count, quat = sim.get_imu_misalignment_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_allclose(quat.cpu().numpy(), _law(TILT, g, expect), atol=2e-6)
    init = torch.zeros((n, _abi.INIT_DIM), device="cuda")
    init[:, 2] = 0.6
    init[:, 3] = 1.0
    sim.reset(init_state=init)
    expect += 1
    count, quat = sim.get_imu_misalignment_state()
    np.testing.assert_array_equal(count.cpu().numpy(), expect)
    np.testing.assert_allclose(quat.cpu().numpy(), _law(TILT, g, expect), atol=2e-6)
    np.testing.assert_allclose(np.linalg.norm(quat.cpu().numpy(), axis=1), 1.0, atol=1e-6)


def test_chunked_host_steps_match_the_device_step(model, torch, monkeypatch):
    """step_host(compact=True, final_obs=True, final_state=True) on five chunks against the same actions through
    upkie_b200_step with compact rows on device buffers (the same kernel in one launch): observations, flags, final
    rows, final and current spine observations bit for bit, and the misalignment state, which follows the law"""
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
        s.set_servo_dropout(0.0, 0.0)
        s.set_imu_misalignment(*TILT)
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
    assert resets[::8192].all() and resets.mean() > 0.5  # resets in every chunk
    for u, v in zip(host.get_imu_misalignment_state(), dev.get_imu_misalignment_state()):
        assert _bits(u.cpu().numpy()) == _bits(v.cpu().numpy())
    count, quat = host.get_imu_misalignment_state()
    count = count.cpu().numpy().astype(np.int64)
    assert count.max() > 2
    g = off + np.arange(n, dtype=np.uint64)
    np.testing.assert_allclose(quat.cpu().numpy(), _law(TILT, g, count), atol=2e-6)


def test_shards_reproduce_the_batch(model, torch):
    n, T = 1024, 30
    whole = _sim(model, _config(), n, SAME_STEP, tilt=TILT)
    half = n // 2
    shards = [_sim(model, _config(), half, SAME_STEP, tilt=TILT, env_offset=o) for o in (0, half)]
    for k in range(T):
        a = _action(torch, model, "gyropod", n, k)
        out = _step(whole, "gyropod", a)
        for s, o in zip(shards, (0, half)):
            part = _step(s, "gyropod", a[o:o + half].contiguous())
            assert _bits(part[0]) == _bits(out[0][o:o + half]), k
            assert _bits(part[5]) == _bits(out[5][o:o + half]), k
    for s, o in zip(shards, (0, half)):
        for x, y in zip(s.get_imu_misalignment_state(), whole.get_imu_misalignment_state()):
            assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy()[o:o + half])


# ---- 6. composition -----------------------------------------------------------------------------------------------------


@pytest.mark.parametrize("kind", ["servos", "gyropod"])
def test_composition(model, torch, kind):
    n, T = 512, 50
    acc_bias, gyro_bias = np.array([0.3, -0.2, 0.1]), np.array([0.02, -0.01, 0.03])
    cfg = _config(max_episode_steps=13, nb_substeps=5)
    for j in range(3):
        cfg.imu_accelerometer_bias[j] = acc_bias[j]
        cfg.imu_gyroscope_bias[j] = gyro_bias[j]
    push = _abi.UpkiePushRandomization(0, 2, 6, 1, 3, (-20.0, -20.0, 0.0), (20.0, 20.0, 0.0))
    sims = []
    for tilt in (TILT, None):
        s = _sim(model, cfg, n, SAME_STEP, tilt=tilt, sense=(1, 4), drop=(0.3, 0.3))
        s.set_action_delay(1, 3)
        s.set_push_randomization(push)
        s.reset(seed=SEED)
        sims.append(s)
    sim, twin = sims
    bias = (np.asarray(acc_bias, dtype=np.float32), np.asarray(gyro_bias, dtype=np.float32))
    resets = 0
    for k in range(T):
        e_old = _quat(sim)
        a = _action(torch, model, kind, n, k)
        x = _step(sim, kind, a, same_step=True)
        y = _step(twin, kind, a, same_step=True)
        e = _quat(sim)
        assert _bits(_state(sim)) == _bits(_state(twin)), k
        assert _bits(x[1]) == _bits(y[1]) and _bits(x[2]) == _bits(y[2]), k
        assert _bits(x[5][:, UNTOUCHED]) == _bits(y[5][:, UNTOUCHED]), k  # the dropouts' latched servos included
        check_spine(x[5], tilt_spine(y[5], e, bias), str(k))  # the delayed snapshot read through e
        check_history(x[6], y[6], e, str(k))
        if kind == "gyropod":
            check_gyropod(x[0], y[5], e, kind, str(k))
        done = (x[1] | x[2]).astype(bool)
        resets += int(done.sum())
        if done.any():
            check_spine(x[4][done], tilt_spine(y[4][done], e_old[done], bias), f"final {k}")
    assert resets > 0


# ---- 7. BaseVelocity --------------------------------------------------------------------------------------------------


def test_base_velocity_mpc_reads_the_sensed_pitch(torch):
    from upkie_b200.base_velocity import mpc_inputs_from_spine
    from upkie_b200.envs import B200VectorEnv

    n = 64
    envs = [B200VectorEnv(n, env_type="base_velocity", autoreset_mode="next_step", imu_misalignment=m)
            for m in ({"pitch": 0.05}, None)]
    for env in envs:
        env.reset(seed=3)
    moved = False
    for k in range(20):
        a = np.tile(np.array([[0.2, 0.0]], dtype=np.float32), (n, 1))
        for env in envs:
            env.step(a)
        x, y = (mpc_inputs_from_spine(env._spine)[0].cpu().numpy() for env in envs)
        # the MPC input of the misaligned env is its own state's pitch + 0.05 (both wheels on the floor)
        tx = envs[0].sim.spine_obs().cpu().numpy()
        np.testing.assert_allclose(x[:, 1], tx[:, _abi.SP_PITCH], atol=0)
        state = envs[0].sim.get_state().cpu().numpy()
        q = state[:, _abi.ST_QUAT:_abi.ST_QUAT + 4]
        true_pitch = np.arcsin(np.clip(2 * (q[:, 0] * q[:, 2] - q[:, 3] * q[:, 1]), -1, 1))
        np.testing.assert_allclose(x[:, 1] - true_pitch, 0.05, atol=3e-3)
        moved |= not np.allclose(x, y)
    assert moved


# ---- 8. checkpoints -----------------------------------------------------------------------------------------------------


def test_checkpoint_round_trip(model, torch):
    from upkie_b200.sim import UpkieSim

    n = 256
    cfg = _config()
    sim = _sim(model, cfg, n, SAME_STEP, tilt=TILT)
    for k in range(10):
        _step(sim, "gyropod", _action(torch, model, "gyropod", n, k), same_step=True)
    sd = sim.state_dict()
    assert sd["imu_misalignment"] == tuple((np.float32(a), np.float32(b)) for a, b in TILT)
    ref = [_step(sim, "gyropod", _action(torch, model, "gyropod", n, 10 + k), same_step=True) for k in range(15)]
    other = UpkieSim(n, model=model, config=cfg)
    other.load_state_dict(sd)
    for k in range(15):
        for x, y in zip(_step(other, "gyropod", _action(torch, model, "gyropod", n, 10 + k), same_step=True), ref[k]):
            if x is not None:
                assert _bits(x) == _bits(y), k
    for x, y in zip(other.get_imu_misalignment_state(), sim.get_imu_misalignment_state()):
        assert _bits(x.cpu().numpy()) == _bits(y.cpu().numpy())
    # a checkpoint without a misalignment turns it off
    del sd["imu_misalignment"]
    other.load_state_dict(sd)
    assert other.imu_misalignment_spec is None


def test_fixed_offsets_and_unit_check(model, torch):
    n = 128
    cfg = _config(max_episode_steps=0)
    sim = _sim(model, cfg, n, 0, tilt=((0.0, 0.0),) * 3, history=None)
    twin = _sim(model, cfg, n, 0, history=None)
    e = quat_np(np.random.default_rng(2).uniform(-0.3, 0.3, (n, 3))).astype(np.float32)
    count = torch.full((n,), 4, dtype=torch.int32, device="cuda")
    sim.set_imu_misalignment_state(count, torch.from_numpy(e).cuda())
    check_spine(sim.spine_obs().cpu().numpy(), tilt_spine(twin.spine_obs().cpu().numpy(), e))
    check_gyropod(sim.reset_obs(6).cpu().numpy(), twin.spine_obs().cpu().numpy(), e, "gyropod")
    bad = torch.from_numpy(e).cuda()
    bad[7] *= 1.001
    with pytest.raises((UpkieException, UpkieRuntimeError), match="unit"):
        sim.set_imu_misalignment_state(count, bad)
    np.testing.assert_allclose(_quat(sim), e, atol=0)  # the rejected state was not taken


# ---- 9. rejections, disabling -------------------------------------------------------------------------------------------


def test_rejections_and_none(model, torch):
    from upkie_b200.envs import B200VectorEnv
    from upkie_b200.sim import UpkieSim

    n = 64
    sim = _sim(model, _config(), n, NEXT_STEP, tilt=TILT, history=None, drop=None)
    for bad, what in ((((0.1, 0.0), (0, 0), (0, 0)), "low <= high"), (((0, 0), (0.0, 0.9), (0, 0)), "pi/4"),
                      (((0, 0), (0, 0), (float("nan"), 0.0)), "finite")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_imu_misalignment(*bad)
    assert sim.imu_misalignment_spec[0] == (np.float32(-0.05), np.float32(0.05))  # the previous spec is kept
    for field, value, what in (("joint_limits", 0, "joint_limits"), ("body_contacts", 1, "body_contacts")):
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            sim.set_config(_config(**{field: value}))
        other = UpkieSim(n, model=model, config=_config(**{field: value}))
        with pytest.raises((UpkieException, UpkieRuntimeError), match=what):
            other.set_imu_misalignment(*TILT)
    spine = UpkieSim(n, model=model, config=_config(spine_mode=1))
    with pytest.raises((UpkieException, UpkieRuntimeError), match="spine_mode"):
        spine.set_imu_misalignment(*TILT)
    with pytest.raises(UpkieException, match="imu_misalignment"):
        B200VectorEnv(8, env_type="gyropod", imu_misalignment={"pitch": (0.2, 0.1)})
    # None: the handle returns to the family it runs without the feature, and its outputs are a plain twin's
    for k in range(3):
        sim.step_gyropod(_action(torch, model, "gyropod", n, k))
    sim.set_imu_misalignment(None)
    assert sim.imu_misalignment_spec is None
    with pytest.raises(UpkieException, match="no IMU misalignment"):
        sim.get_imu_misalignment_state()
    plain = UpkieSim(n, model=model, config=_config())
    plain.set_autoreset(NEXT_STEP, SEED, 0)
    plain.load_state_dict(sim.state_dict())
    for k in range(20):
        a = _action(torch, model, "gyropod", n, 3 + k)
        x, y = sim.step_gyropod(a), plain.step_gyropod(a)
        for u, v in zip(x, y):
            assert _bits(u.cpu().numpy()) == _bits(v.cpu().numpy()), k
        assert _bits(sim.spine_obs().cpu().numpy()) == _bits(plain.spine_obs().cpu().numpy()), k


@pytest.mark.parametrize("env_type", ["servos", "gyropod", "pendulum", "base_velocity"])
def test_vector_env(torch, env_type):
    from upkie_b200 import make_vec

    env = make_vec("Upkie-B200-" + {"servos": "Servos", "gyropod": "Gyropod", "pendulum": "Pendulum",
                                     "base_velocity": "BaseVelocity"}[env_type], 64,
                   imu_misalignment={"roll": (-0.01, 0.01), "pitch": (-0.03, 0.03)})
    env.reset(seed=3)
    count, quat = env.sim.get_imu_misalignment_state()
    assert (count.cpu().numpy() == 1).all()
    spec = ((-0.01, 0.01), (-0.03, 0.03), (0.0, 0.0))
    np.testing.assert_allclose(quat.cpu().numpy(), _law(spec, np.arange(64, dtype=np.uint64), np.ones(64, np.int64), seed=3),
                               atol=2e-6)
    for _ in range(5):
        env.step(env.action_space.sample())
    env.set_imu_misalignment(None)
    env.step(env.action_space.sample())
