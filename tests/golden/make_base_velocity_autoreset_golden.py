#!/usr/bin/env python
# SPDX-License-Identifier: Apache-2.0
"""Golden runs of the reference's OWN UpkieBaseVelocity env under Gymnasium's two auto-reset modes, on the oracle.

Run in the build container:  python tests/golden/make_base_velocity_autoreset_golden.py

Same stand-ins and OracleBackend as make_base_velocity_golden.py. The unmodified UpkieBaseVelocity class is driven by
two hand-written vector-env loops with a short time limit (TimeLimit semantics: truncated once T steps have run since
the last reset), so that every run holds several episodes:
  - next_step: the step after an env ended (terminated | truncated) ignores its action and calls env.reset()
    instead, returning the reset observation with reward 0 and both flags False; that step is not counted;
  - same_step: the step in which an env ends calls env.reset() at once and returns the reset observation with the
    flags set; the observation it reached is the final observation.
The initial state carries no randomisation, so every episode starts from the nominal state (as the device sampler
of the fused auto-resets does). Output: tests/golden/base_velocity_autoreset_runs.json, replayed by
tests/test_base_velocity_post.py (CPU, base_velocity_tick on the oracle) and tests/test_gpu_base_velocity_autoreset.py
(B200VectorEnv in both modes).
"""
import importlib.util
import json
import os
import sys
import types

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
OUT = os.path.join(HERE, "base_velocity_autoreset_runs.json")
sys.path.insert(0, HERE)

TIME_LIMIT = 40
TICKS = 200


def make_env():
    import make_mpc_golden as mg
    import make_wrapper_golden as wg

    wg.install_fake_gymnasium()
    mg.install_stand_ins()
    envs = wg.load_reference()
    ctrl = types.ModuleType("upkie.controllers")
    ctrl.__path__ = [os.path.join(wg.REF, "upkie", "controllers")]
    sys.modules["upkie.controllers"] = ctrl
    spec = importlib.util.spec_from_file_location("upkie.controllers.mpc_balancer",
                                                  os.path.join(wg.REF, "upkie/controllers/mpc_balancer.py"))
    mb = importlib.util.module_from_spec(spec)
    sys.modules["upkie.controllers.mpc_balancer"] = mb
    spec.loader.exec_module(mb)
    spec = importlib.util.spec_from_file_location("upkie.envs.upkie_base_velocity",
                                                  os.path.join(wg.REF, "upkie/envs/upkie_base_velocity.py"))
    bv = importlib.util.module_from_spec(spec)
    sys.modules["upkie.envs.upkie_base_velocity"] = bv
    spec.loader.exec_module(bv)

    import tempfile

    from oracle import oracle as O
    from upkie_b200 import _abi
    from upkie_b200.envs import spine_row_to_dict
    from upkie_b200.model import Model as B200Model
    from upkie_b200.urdf import write_urdf
    from upkie_b200.wire import action_dict_to_row

    Backend = sys.modules["upkie.envs.backends"].Backend
    RefModel = sys.modules["upkie.model"].Model
    RobotState = sys.modules["upkie.utils.robot_state"].RobotState
    b200_model = B200Model.standard_upkie()
    urdf_path = os.path.join(tempfile.mkdtemp(), "robot.urdf")
    write_urdf(b200_model, urdf_path, split_fixed_links=True)
    ref_model = RefModel(urdf_path)

    class OracleBackend(Backend):
        def __init__(self):
            self.cfg = _abi.default_sim_config()
            self.cfg.skip_action_clamps = 1
            self.sim = O.OracleSim(b200_model, self.cfg, 1, threads=1)

        def close(self):
            pass

        def get_spine_observation(self):
            return spine_row_to_dict(self.sim.spine_obs()[0])

        def reset(self, init_state):
            row = np.zeros((1, _abi.INIT_DIM))
            row[0, 0:3] = init_state.position_base_in_world
            q = init_state.orientation_base_in_world.as_quat()
            row[0, 3:7] = [q[3], q[0], q[1], q[2]]
            row[0, 7:10] = init_state.linear_velocity_base_to_world_in_world
            row[0, 10:13] = init_state.angular_velocity_base_in_base
            row[0, 13:19] = init_state.joint_configuration
            self.init_row = row.copy()
            self.sim.reset(row)
            return self.get_spine_observation()

        def step(self, action):
            a = action_dict_to_row(action).astype(np.float64)
            self.sim.step_servos(a.reshape(1, 6, 6))
            return self.get_spine_observation()

    backend = OracleBackend()
    init = RobotState(position_base_in_world=np.array([0.0, 0.0, 0.58]))  # no randomisation: nominal episodes
    servos = envs["upkie_servos"].UpkieServos(backend=backend, frequency=200.0, frequency_checks=False, init_state=init,
                                               regulate_frequency=False, model=ref_model)
    return bv.UpkieBaseVelocity(servos), backend


def actions():
    rng = np.random.default_rng(20261016)
    out, v, w = [], 0.0, 0.0
    for t in range(TICKS):
        if t % 25 == 0:
            v, w = float(rng.uniform(-0.4, 0.4)), float(rng.uniform(-0.8, 0.8))
        out.append(np.array([v, w], dtype=np.float32))
    return out


def run(mode):
    env, backend = make_env()
    obs, _ = env.reset(seed=1)
    rec = {"init_row": backend.init_row[0].tolist(), "actions": [], "obs": [], "terminated": [], "truncated": [],
           "final_obs": [], "commanded_velocity": []}
    elapsed, pending = 0, False
    for act in actions():
        final = None
        if mode == "next_step" and pending:
            obs, _ = env.reset()
            reward, terminated, truncated = 0.0, False, False
            elapsed = 0
        else:
            obs, reward, terminated, _, _ = env.step(act)
            elapsed += 1
            truncated = elapsed >= TIME_LIMIT
            if mode == "same_step" and (terminated or truncated):
                final = [float(x) for x in obs]
                obs, _ = env.reset()
                elapsed = 0
        pending = terminated or truncated
        assert reward == 0.0
        rec["actions"].append([float(x) for x in act])
        rec["obs"].append([float(x) for x in obs])
        rec["terminated"].append(bool(terminated))
        rec["truncated"].append(bool(truncated))
        rec["final_obs"].append(final)
        rec["commanded_velocity"].append(float(env.mpc_balancer.commanded_velocity))
    return rec


def main():
    runs = {"generator": "tests/golden/make_base_velocity_autoreset_golden.py", "time_limit": TIME_LIMIT,
            "next_step": run("next_step"), "same_step": run("same_step")}
    for mode in ("next_step", "same_step"):
        r = runs[mode]
        print(mode, "terminated", sum(r["terminated"]), "truncated", sum(r["truncated"]))
    with open(OUT, "w") as f:
        json.dump(runs, f)
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KB")


if __name__ == "__main__":
    main()
