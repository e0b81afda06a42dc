#!/usr/bin/env python3
# SPDX-License-Identifier: Apache-2.0
"""Offline parity audit against a REAL PyBullet: record the same open-loop run on two backends, compare.

The contact phase of the simulation restates Bullet (third-party, absent from the build container), so its parity
is unpinned (DESIGN.md section 5). This tool closes that gap on any machine that has ``upkie`` + ``pybullet``
installed: both ``upkie_b200.backend.B200Backend`` and the reference's ``PyBulletBackend`` implement the same
backend interface (``reset(init_state) -> observation``, ``step(action) -> observation``;
``upkie/envs/backends/backend.py:11-50``), so the same seeded action sequence is fed to each and the spine
observations are compared tick by tick.

    # on a GPU machine
    python tools/parity_audit.py record --backend b200 --scenario stand --ticks 400 --out b200.mpack
    # on a machine with `pip install upkie pybullet upkie_description`
    python tools/parity_audit.py record --backend pybullet --scenario stand --ticks 400 --out bullet.mpack
    # anywhere
    python tools/parity_audit.py compare b200.mpack bullet.mpack

Files are msgpack streams in the reference's own serialisation (``upkie_b200/wire.py``): one header dictionary, then
one ``{"tick", "action", "observation"}`` dictionary per tick. Scenarios are open loop on purpose (the actions do not
depend on the observations), so that both backends receive bit-identical inputs:

  stand     legs held at zero by the position controller, wheels velocity-controlled along a slow sine
  squat     hips / knees follow a slow squat, wheels as above
  torques   seeded random feedforward torques on every joint (kp = kd = 0), from a 1 m drop
  fall      no action at all from an initial pitch of 0.4 rad: the robot topples and comes to rest on whatever collision
            shapes its links carry (body-ground contact rows, DESIGN.md section 3; compare the resting base height and pitch)

    # on the machine with a real pybullet: the third-party constants this repo restates from memory, next to Bullet's own
    python tools/parity_audit.py constants [--urdf upkie.urdf]

Differences to expect: the stand-in inertias of ``Model.standard_upkie()`` (pass ``--urdf`` with the real
``upkie_description`` URDF on the B200 side to remove them), Bullet's up-to-four-point tire manifold against one point
here, and chaotic divergence after a touchdown.
"""
import argparse
import os
import sys

import msgpack
import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

JOINTS = ("left_hip", "left_knee", "left_wheel", "right_hip", "right_knee", "right_wheel")
SCENARIOS = ("stand", "squat", "torques", "fall")


def scenario_actions(name: str, ticks: int, dt: float, seed: int, tau_max) -> list:
    """The open-loop action dictionaries of a scenario (``PyBulletBackend.step`` contract,
    ``pybullet_backend.py:276-300``)."""
    rng = np.random.default_rng(seed)
    actions = []
    for k in range(ticks):
        t = k * dt
        if name == "fall":
            actions.append({})  # step(action={}) is legal = no torques (tests/envs/backends/test_pybullet_backend.py:28-31)
            continue
        servo = {}
        wheel_velocity = 2.0 * np.sin(2.0 * np.pi * 0.5 * t)  # rad/s
        squat = 0.3 * (1.0 - np.cos(2.0 * np.pi * 0.5 * t)) if name == "squat" else 0.0
        for j, joint in enumerate(JOINTS):
            side = 1.0 if joint.startswith("left") else -1.0
            if name == "torques":
                servo[joint] = {
                    "position": float("nan"), "velocity": 0.0, "kp_scale": 0.0, "kd_scale": 0.0,
                    "feedforward_torque": float(rng.uniform(-0.3, 0.3) * tau_max[j]),
                    "maximum_torque": float(tau_max[j]),
                }
            elif joint.endswith("wheel"):
                servo[joint] = {
                    "position": float("nan"), "velocity": float(side * wheel_velocity), "kp_scale": 1.0,
                    "kd_scale": 1.0, "feedforward_torque": 0.0, "maximum_torque": float(tau_max[j]),
                }
            else:
                target = squat if joint.endswith("hip") else -2.0 * squat
                servo[joint] = {
                    "position": float(side * target), "velocity": 0.0, "kp_scale": 1.0, "kd_scale": 1.0,
                    "feedforward_torque": 0.0, "maximum_torque": float(tau_max[j]),
                }
        actions.append({"servo": servo})
    return actions


def make_backend(kind: str, dt: float, urdf: str = None):
    """(backend, RobotState class, tau_max[6]) for ``b200`` or ``pybullet``."""
    if kind == "b200":
        from upkie_b200.backend import B200Backend
        from upkie_b200.model import Model
        from upkie_b200.robot_state import RobotState

        model = Model.from_urdf(urdf) if urdf else Model.standard_upkie()
        return B200Backend(dt=dt, model=model), RobotState, [float(x) for x in model.tau_max]
    if kind == "pybullet":
        from upkie.envs.backends.pybullet_backend import PyBulletBackend  # the reference, unmodified
        from upkie.model import Model
        from upkie.utils.robot_state import RobotState

        model = Model(urdf) if urdf else Model()
        tau_max = [float(joint.limit.effort) for joint in model.joints]
        return PyBulletBackend(dt=dt, gui=False, model=model), RobotState, tau_max
    raise SystemExit(f"unknown backend {kind!r}")


def flatten(prefix: str, value, out: dict) -> None:
    """Nested observation dictionary -> {"a.b.c": float array}; non-numeric leaves are dropped."""
    if isinstance(value, dict):
        for key, sub in value.items():
            flatten(f"{prefix}.{key}" if prefix else str(key), sub, out)
        return
    try:
        arr = np.asarray(value, dtype=float).ravel()
    except (TypeError, ValueError):
        return
    if arr.size:
        out[prefix] = arr


def record(backend, robot_state_cls, actions: list, header: dict, out_path: str) -> None:
    from upkie_b200 import wire

    height = 1.0 if header["scenario"] == "torques" else 0.6
    kwargs = {}
    if header["scenario"] == "fall":
        from scipy.spatial.transform import Rotation

        kwargs["orientation_base_in_world"] = Rotation.from_euler("y", 0.4)
    init = robot_state_cls(position_base_in_world=np.array([0.0, 0.0, height]), **kwargs)
    with open(out_path, "wb") as f:
        f.write(wire.pack_dict(header))
        observation = backend.reset(init)
        f.write(wire.pack_dict({"tick": 0, "action": {}, "observation": observation}))
        for k, action in enumerate(actions):
            observation = backend.step(action)
            f.write(wire.pack_dict({"tick": k + 1, "action": action, "observation": observation}))


def load(path: str):
    unpacker = msgpack.Unpacker(raw=False, strict_map_key=False)
    with open(path, "rb") as f:
        unpacker.feed(f.read())
    records = list(unpacker)
    return records[0], records[1:]


def compare(path_a: str, path_b: str, checkpoints=(1, 2, 5, 10, 20, 50, 100, 200, 400, 1000)) -> dict:
    """Per observation key: max |difference| up to each checkpoint tick. Returns {key: {tick: value}}."""
    header_a, rec_a = load(path_a)
    header_b, rec_b = load(path_b)
    for key in ("scenario", "seed", "dt"):
        if header_a.get(key) != header_b.get(key):
            raise SystemExit(f"the two recordings differ in {key}: {header_a.get(key)} vs {header_b.get(key)}")
    n = min(len(rec_a), len(rec_b))
    table, running = {}, {}
    for k in range(n):
        fa, fb = {}, {}
        flatten("", rec_a[k]["observation"], fa)
        flatten("", rec_b[k]["observation"], fb)
        for key in fa.keys() & fb.keys():
            if fa[key].shape != fb[key].shape:
                continue
            with np.errstate(invalid="ignore"):
                d = float(np.nanmax(np.abs(fa[key] - fb[key]))) if fa[key].size else 0.0
            running[key] = max(running.get(key, 0.0), d)
        tick = rec_a[k]["tick"]
        if tick in checkpoints or k == n - 1:
            for key, value in running.items():
                table.setdefault(key, {})[tick] = value
    return table


def print_table(table: dict) -> None:
    ticks = sorted({t for row in table.values() for t in row})
    print(f"{'max |difference| up to tick':48s}" + "".join(f"{t:>10d}" for t in ticks))
    for key in sorted(table):
        print(f"{key:48s}" + "".join(f"{table[key].get(t, float('nan')):10.2e}" for t in ticks))


# what UpkieSimConfig restates from memory of Bullet / PyBullet -> the key of pybullet.getPhysicsEngineParameters()
# (or of getDynamicsInfo of a link) that holds the real value
RESTATED_CONSTANTS = (
    ("pgs_iterations", "numSolverIterations", "physics"),
    ("solver_residual_threshold", "solverResidualThreshold", "physics"),
    ("contact_breaking_threshold", "contactBreakingThreshold", "physics"),
    ("body_contact_erp", "contactERP", "physics"),
    ("joint_limit_erp", "erp", "physics"),
    ("warmstarting_factor", "warmStartingFactor", "physics"),
    ("linear_damping", "linearDamping", "dynamics"),
    ("angular_damping", "angularDamping", "dynamics"),
    ("contact_stiffness", "contactStiffness", "dynamics:left_wheel_tire"),
    ("contact_damping", "contactDamping", "dynamics:left_wheel_tire"),
    ("body_friction", "lateralFriction", "dynamics:torso"),
)


def constants_report(our_config, physics: dict, dynamics: dict) -> list:
    """Rows ``(field of UpkieSimConfig, value here, PyBullet key, value there or None)``. ``physics`` is the dictionary
    ``pybullet.getPhysicsEngineParameters()`` returns, ``dynamics`` maps a link name ("" = any) to a dictionary of the
    named entries of ``pybullet.getDynamicsInfo`` (lateralFriction, contactStiffness, contactDamping, linearDamping...)."""
    rows = []
    for field, key, where in RESTATED_CONSTANTS:
        ours = getattr(our_config, field)
        if where == "physics":
            theirs = physics.get(key)
        else:
            link = where.split(":", 1)[1] if ":" in where else ""
            theirs = (dynamics.get(link) or dynamics.get("") or {}).get(key)
        rows.append((field, float(ours), key, None if theirs is None else float(theirs)))
    return rows


def pybullet_constants(urdf: str = None):
    """Load plane + robot in a DIRECT PyBullet like ``PyBulletBackend.__init__`` does (``pybullet_backend.py:100-125``:
    no solver parameter is changed) and read the constants back."""
    import pybullet
    import pybullet_data

    if urdf is None:
        import upkie_description

        urdf = upkie_description.URDF_PATH
    client = pybullet.connect(pybullet.DIRECT)
    pybullet.setAdditionalSearchPath(pybullet_data.getDataPath())
    pybullet.loadURDF("plane.urdf")
    robot = pybullet.loadURDF(urdf, basePosition=[0, 0, 0.6])
    physics = dict(pybullet.getPhysicsEngineParameters())
    names = ("mass", "lateralFriction", "localInertiaDiagonal", "localInertialPos", "localInertialOrn", "restitution",
             "rollingFriction", "spinningFriction", "contactDamping", "contactStiffness", "bodyType", "collisionMargin")
    dynamics = {}
    for idx in range(-1, pybullet.getNumJoints(robot)):
        link = "base" if idx < 0 else pybullet.getJointInfo(robot, idx)[12].decode()
        info = pybullet.getDynamicsInfo(robot, idx)
        dynamics[link] = {k: v for k, v in zip(names, info) if isinstance(v, (int, float))}
        shapes = pybullet.getCollisionShapeData(robot, idx)
        dynamics[link]["collisionShapes"] = len(shapes)
    dynamics[""] = dynamics.get("base", {})
    pybullet.disconnect(client)
    return physics, dynamics


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    sub = ap.add_subparsers(dest="cmd", required=True)
    rec = sub.add_parser("record")
    rec.add_argument("--backend", choices=("b200", "pybullet"), required=True)
    rec.add_argument("--scenario", choices=SCENARIOS, default="stand")
    rec.add_argument("--ticks", type=int, default=400)
    rec.add_argument("--frequency", type=float, default=200.0)
    rec.add_argument("--seed", type=int, default=0)
    rec.add_argument("--urdf", default=None, help="robot description to load on this side (default: the backend's own)")
    rec.add_argument("--out", required=True)
    cmp_ = sub.add_parser("compare")
    cmp_.add_argument("a")
    cmp_.add_argument("b")
    con = sub.add_parser("constants", help="print the Bullet / PyBullet constants restated in UpkieSimConfig next to a real PyBullet's")
    con.add_argument("--urdf", default=None)
    args = ap.parse_args(argv)
    if args.cmd == "constants":
        from upkie_b200 import _abi

        physics, dynamics = pybullet_constants(args.urdf)
        print(f"{'UpkieSimConfig field':32s}{'here':>14s}  {'PyBullet':28s}{'there':>14s}")
        for field, ours, key, theirs in constants_report(_abi.default_sim_config(), physics, dynamics):
            there = "n/a" if theirs is None else f"{theirs:.6g}"
            flag = "" if theirs is None or abs(theirs - ours) <= 1e-9 + 1e-6 * abs(ours) else "   <-- differs"
            print(f"{field:32s}{ours:14.6g}  {key:28s}{there:>14s}{flag}")
        links = sorted(k for k, v in dynamics.items() if k and v.get("collisionShapes"))
        print("links with collision shapes:", ", ".join(links) or "none")
        return 0
    if args.cmd == "record":
        dt = 1.0 / args.frequency
        backend, robot_state_cls, tau_max = make_backend(args.backend, dt, args.urdf)
        actions = scenario_actions(args.scenario, args.ticks, dt, args.seed, tau_max)
        header = {"format": "upkie_b200.parity_audit/1", "backend": args.backend, "scenario": args.scenario,
                  "seed": args.seed, "dt": dt, "ticks": args.ticks, "urdf": args.urdf or ""}
        record(backend, robot_state_cls, actions, header, args.out)
        backend.close()
        print(f"wrote {args.out}: {args.ticks} ticks of scenario '{args.scenario}' on backend '{args.backend}'")
        return 0
    print_table(compare(args.a, args.b))
    return 0


if __name__ == "__main__":
    sys.exit(main())
