# SPDX-License-Identifier: Apache-2.0
"""GPU parity: sm_90a kernels (through the C ABI) vs the fp64 CPU oracle."""
import numpy as np
import pytest

from conftest import random_servo_actions, random_states

pytestmark = pytest.mark.gpu

# fp32 kernels vs fp64 oracle after one 5 ms tick from identical states.
# Velocities carry the touchdown sensitivity of the Bullet-style contact row
# (d v / d penetration = 1/h = 1000 1/s, times 1/r = 20 on wheel rates), so the
# worst-case velocity tolerance is looser than the position tolerance.
# Round 2: the worst-case caps are tied to what the fp64 -> fp32 change alone costs, measured on the same inputs with
# the oracle instantiated in fp32 (textbook link-frame ABA): on these 2 048 states the fp32 oracle's worst joint-rate
# error is 1.1e-3 rad/s (base twist 3.6e-5), the kernels' arithmetic compiled for the host 2.2e-3 (7.3e-5). Round 1
# allowed 0.4 rad/s here. The measured values are appended to the JSON file named by UPKIE_PARITY_REPORT, if set.
TOL_POS = 2e-5
TOL_VEL_STEADY = 5e-4
TOL_VEL_WORST = 1e-3        # base twist, worst env
TOL_JOINT_RATE_WORST = 2e-2  # joint rates, worst env (touchdown sensitivity x 1/r on wheel rates)


def _report(name, **values):
    import json
    import os

    path = os.environ.get("UPKIE_PARITY_REPORT")
    if not path:
        return
    try:
        data = json.load(open(path)) if os.path.exists(path) else {}
    except Exception:
        data = {}
    data[name] = {k: float(v) for k, v in values.items()}
    with open(path, "w") as f:
        json.dump(data, f, indent=1)


def _mk(n, model, cfg=None):
    import torch

    from upkie_b200 import _abi
    from upkie_b200.sim import UpkieSim

    cfg = cfg if cfg is not None else _abi.default_sim_config()
    return UpkieSim(n, model=model, config=cfg), cfg, torch


def test_one_tick_servos_matches_oracle(model, oracle_lib):
    n = 2048
    sim, cfg, torch = _mk(n, model)
    st = random_states(n, seed=3)
    act = random_servo_actions(n, model, seed=4)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
    st32 = st.astype(np.float32)
    osim.set_state(st32.astype(np.float64))
    sim.set_state(torch.from_numpy(st32).cuda())
    act32 = act.astype(np.float32)
    oobs, orew, oterm, otrunc = osim.step_servos(act32.astype(np.float64))
    gobs, grew, gterm, gtrunc = sim.step_servos(torch.from_numpy(act32).cuda())
    torch.cuda.synchronize()
    gs = sim.get_state().cpu().numpy().astype(np.float64)
    os_ = osim.get_state()
    dpos = np.abs(gs[:, :7] - os_[:, :7]).max()
    dq = np.abs(gs[:, 13:19] - os_[:, 13:19]).max()
    dvel = np.abs(gs[:, 7:13] - os_[:, 7:13])
    dqd = np.abs(gs[:, 19:25] - os_[:, 19:25])
    assert dpos < TOL_POS and dq < 2e-4, (dpos, dq)
    assert np.median(dvel.max(axis=1)) < TOL_VEL_STEADY
    assert np.median(dqd.max(axis=1)) < TOL_VEL_STEADY
    # the same tick on the oracle in fp32: what single precision alone costs on these inputs
    o32 = oracle_lib.OracleSim(model, cfg, n, use_float=True, threads=8)
    o32.set_state(st32.astype(np.float64))
    o32.step_servos(act32.astype(np.float64))
    s32 = o32.get_state()
    dvel32, dqd32 = np.abs(s32[:, 7:13] - os_[:, 7:13]).max(), np.abs(s32[:, 19:25] - os_[:, 19:25]).max()
    _report("one_tick_servos_2048", base_twist_worst=dvel.max(), joint_rate_worst=dqd.max(),
            joint_rate_p99=np.percentile(dqd.max(axis=1), 99), joint_rate_median=np.median(dqd.max(axis=1)),
            fp32_oracle_base_twist_worst=dvel32, fp32_oracle_joint_rate_worst=dqd32, position_worst=dpos, joint_angle_worst=dq)
    assert dvel.max() < TOL_VEL_WORST and dqd.max() < TOL_JOINT_RATE_WORST, (dvel.max(), dqd.max())
    assert dqd.max() < max(10.0 * dqd32, 5e-3), (dqd.max(), dqd32)  # within an order of magnitude of fp32 itself
    assert np.percentile(dqd.max(axis=1), 99) < 1e-3
    # observations: positions/velocities/torques as the state, constants exact
    g = gobs.cpu().numpy().astype(np.float64)
    assert np.array_equal(g[:, :, 3], np.full((n, 6), 42.0))
    assert np.array_equal(g[:, :, 4], np.full((n, 6), 18.0))
    assert np.abs(g[:, :, 0] - oobs[:, :, 0]).max() < 2e-4
    assert np.median(np.abs(g[:, :, 2] - oobs[:, :, 2])) < 1e-3
    # integer outputs bit-exact
    assert np.array_equal(gterm.cpu().numpy(), oterm)
    assert np.array_equal(gtrunc.cpu().numpy(), otrunc)
    assert np.array_equal(grew.cpu().numpy(), orew.astype(np.float32))
    # error flags (clamped / NaN velocity) bit-exact
    assert np.array_equal(sim.error_flags().cpu().numpy().astype(np.uint32), osim.error_flags())
    assert np.array_equal(gs[:, 40], os_[:, 40])  # floor contact flag


def test_spine_observation_matches_oracle(model, oracle_lib):
    n = 512
    sim, cfg, torch = _mk(n, model)
    st32 = random_states(n, seed=7).astype(np.float32)
    act32 = random_servo_actions(n, model, seed=8).astype(np.float32)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
    osim.set_state(st32.astype(np.float64))
    sim.set_state(torch.from_numpy(st32).cuda())
    osim.step_servos(act32.astype(np.float64))
    sim.step_servos(torch.from_numpy(act32).cuda())
    g = sim.spine_obs().cpu().numpy().astype(np.float64)
    o = osim.spine_obs()
    # quaternion sign convention must match exactly (scipy branch choice)
    assert np.abs(g[:, 16:20] - o[:, 16:20]).max() < 1e-4
    assert np.abs(g[:, 6] - o[:, 6]).max() < 1e-5  # pitch
    assert np.abs(g[:, 7:16] - o[:, 7:16]).max() < 1e-5  # rotation matrix
    assert np.array_equal(g[:, 29], o[:, 29])  # contact
    assert np.median(np.abs(g[:, 23:29] - o[:, 23:29])) < 5e-2  # IMU accelerations (finite differences / dt)
    assert np.abs(g[:, 60] - o[:, 60]).max() < 1e-5  # odometry position
