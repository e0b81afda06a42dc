# SPDX-License-Identifier: Apache-2.0
"""GPU tests of the joint-limit rows on the device (k_step<.., FAM_LIMITS, ..>: config.joint_limits = 1 -> 3 on the
device, 2, 3) against the oracle, the Backend contact query, and the parity-audit recorder.

Written at the end of round 1 (hence the file name: it sorted last so that its first run on a GPU could not mask the
tests that had already been green there). The CPU build of the same kernel code agrees with the oracle
(tests/test_kernel_arithmetic_cpu.py::test_joint_limit_rows)."""
import numpy as np
import pytest

from conftest import at_joint_bounds, random_servo_actions
from upkie_b200 import _abi

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("solver", [1, 2, 3])
def test_joint_limit_rows_on_device(model, oracle_lib, solver):
    """solver 1: scalar slow path for the robots with an active limit row; 2: packed ten-row solver for all."""
    import torch

    from upkie_b200.sim import UpkieSim

    n = 2048
    cfg = _abi.default_sim_config()
    cfg.joint_limits = solver
    sim = UpkieSim(n, model=model, config=cfg)
    cfg_plain = _abi.default_sim_config()
    cfg_plain.joint_limits = 0
    plain = UpkieSim(n, model=model, config=cfg_plain)
    osim = oracle_lib.OracleSim(model, cfg, n, threads=8)
    st = at_joint_bounds(model, n, seed=5)
    act = random_servo_actions(n, model, seed=12).astype(np.float32)
    a = torch.from_numpy(act).cuda()
    sim.set_state(torch.from_numpy(st).cuda())
    plain.set_state(torch.from_numpy(st).cuda())
    osim.set_state(st.astype(np.float64))
    for _ in range(3):
        sim.step_servos(a)
        plain.step_servos(a)
        osim.step_servos(act.astype(np.float64))
        g = sim.get_state().cpu().numpy().astype(np.float64)
        o = osim.get_state()
        d = np.abs(g[:, :25] - o[:, :25])
        assert d[:, :7].max() < 2e-5 and d[:, 13:19].max() < 2e-4
        assert np.median(d[:, 19:25].max(axis=1)) < 5e-5 and np.percentile(d[:, 19:25].max(axis=1), 99) < 2e-3
        assert (g[:, 40] != o[:, 40]).sum() <= 1  # contact flags (one robot may sit within round-off of the threshold)
        assert np.abs(g[:, 19:25] - plain.get_state().cpu().numpy()[:, 19:25]).max() > 5.0  # the rows matter
        osim.set_state(g)
        plain.set_state(sim.get_state())


def test_backend_contact_points_on_device(model):
    """``B200Backend.get_contact_points`` (``PyBulletBackend.get_contact_points``, pybullet_backend.py:660-716) for
    a robot standing on its wheels: two tire contacts that carry its weight, filtered by link name."""
    from upkie_b200.backend import B200Backend
    from upkie_b200.robot_state import RobotState

    backend = B200Backend(dt=1.0 / 200.0)
    backend.reset(RobotState(position_base_in_world=np.array([0.0, 0.0, 0.6])))
    hold = {"servo": {name: {"position": 0.0, "velocity": 0.0, "maximum_torque": float(model.tau_max[j])}
                      for j, name in enumerate(_abi.JOINT_NAMES)}}
    for _ in range(40):
        backend.step(hold)
    contacts = backend.get_contact_points()
    assert [c.link_name for c in contacts] == ["left_wheel_tire", "right_wheel_tire"]
    weight = float(np.sum(model.mass)) * 9.81
    assert abs(sum(c.force_in_world[2] for c in contacts) - weight) < 0.15 * weight
    assert all(abs(c.position_contact_in_world[2]) < 5e-3 for c in contacts)
    assert len(backend.get_contact_points("left_wheel_tire")) == 1
    assert backend.get_contact_points("imu") == [] and backend.get_contact_points("no_such_link") == []
    backend.close()


def test_parity_audit_records_from_the_b200_backend(tmp_path):
    """tools/parity_audit.py record --backend b200: the recording a real-PyBullet machine would be compared with."""
    import importlib.util
    import os

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    spec = importlib.util.spec_from_file_location("parity_audit", os.path.join(root, "tools", "parity_audit.py"))
    audit = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(audit)
    paths = [str(tmp_path / f"run{k}.mpack") for k in range(2)]
    for path in paths:
        assert audit.main(["record", "--backend", "b200", "--scenario", "squat", "--ticks", "30", "--out", path]) == 0
    header, records = audit.load(paths[0])
    assert header["backend"] == "b200" and len(records) == 31
    assert abs(records[-1]["observation"]["servo"]["left_hip"]["position"]) > 1e-3  # the squat moved the hips
    table = audit.compare(paths[0], paths[1])
    assert max(max(row.values()) for row in table.values()) == 0.0  # deterministic: two runs, identical recordings
