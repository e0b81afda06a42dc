# SPDX-License-Identifier: Apache-2.0
"""tools/parity_audit.py: its seeded scenarios and its constants report. The tool's purpose - a run against a REAL
PyBullet - needs a machine that has one."""
import importlib.util
import os

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture()
def audit():
    spec = importlib.util.spec_from_file_location("parity_audit", os.path.join(ROOT, "tools", "parity_audit.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_scenarios_are_open_loop_and_seeded(audit):
    tau_max = [16.0, 16.0, 1.7, 16.0, 16.0, 1.7]
    for name in audit.SCENARIOS:
        a = audit.scenario_actions(name, 50, 0.005, 3, tau_max)
        b = audit.scenario_actions(name, 50, 0.005, 3, tau_max)
        assert repr(a) == repr(b)  # same seed, same actions (NaN positions included)
        if name == "fall":
            assert a == [{}] * 50  # no action: the robot topples onto its collision shapes
            continue
        assert len(a) == 50 and set(a[0]["servo"]) == set(audit.JOINTS)
        for joint, servo in a[7]["servo"].items():
            assert abs(servo["feedforward_torque"]) <= servo["maximum_torque"] and not np.isnan(servo["velocity"])
    assert repr(audit.scenario_actions("torques", 5, 0.005, 1, tau_max)) != repr(
        audit.scenario_actions("torques", 5, 0.005, 2, tau_max))


def test_constants_report_flags_differences(audit):
    """`parity_audit.py constants`: the report logic on a made-up PyBullet answer (a real one needs a machine that has
    pybullet): every restated Bullet constant of UpkieSimConfig is looked up under its PyBullet name."""
    from upkie_b200 import _abi

    cfg = _abi.default_sim_config()
    physics = {"numSolverIterations": 50, "solverResidualThreshold": 1e-7, "contactBreakingThreshold": 0.02,
               "contactERP": 0.2, "erp": 0.2}
    dynamics = {"left_wheel_tire": {"contactStiffness": 30000.0, "contactDamping": 1000.0, "lateralFriction": 1.0},
                "torso": {"lateralFriction": 0.5}, "": {"linearDamping": 0.04, "angularDamping": 0.04}}
    rows = {field: (ours, key, theirs) for field, ours, key, theirs in audit.constants_report(cfg, physics, dynamics)}
    assert rows["solver_residual_threshold"] == (1e-7, "solverResidualThreshold", 1e-7)
    assert rows["pgs_iterations"][2] == 50.0 and rows["contact_stiffness"][2] == 30000.0
    assert rows["warmstarting_factor"][2] is None  # a key this PyBullet did not report
    assert all(theirs is None or abs(theirs - ours) < 1e-9 for ours, _, theirs in rows.values())
    for field, _, _ in audit.RESTATED_CONSTANTS:
        assert hasattr(cfg, field)
