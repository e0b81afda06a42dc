#!/usr/bin/env python3
# SPDX-License-Identifier: Apache-2.0
"""What the body-contact kernel family (NOISE = 4) costs when no torso touches the floor: 4 096 pendulum envs with
body_contacts off / on, device time per tick from a CUDA-graph replay (run on a GPU; prints two lines)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from upkie_b200.envs import B200VectorEnv  # noqa: E402
from upkie_b200.model import Model  # noqa: E402
from upkie_b200.robot_state import RobotState, RobotStateRandomization  # noqa: E402

dev = torch.device("cuda:0")
n = 4096
for on in (False, True):
    gen = torch.Generator(device=dev)
    gen.manual_seed(7)
    env = B200VectorEnv(n, "pendulum", device=0, autoreset_mode="next_step", model=Model.standard_upkie(),
                        init_state=RobotState(randomization=RobotStateRandomization(pitch=0.1)), body_contacts=on)
    env.sim.set_autoreset(1, 2025, 0)
    env.sim.reset(seed=2025)
    acts = [((torch.rand((n, 1), device=dev, generator=gen) * 2 - 1) * 3.0).contiguous() for _ in range(8)]
    for i in range(30):
        env.sim.step_pendulum(acts[i % 8])
    torch.cuda.synchronize()
    s = torch.cuda.Stream(device=dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        for i in range(48):
            env.sim.step_pendulum(acts[i % 8])
    torch.cuda.synchronize()
    g.replay()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(20):
        g.replay()
    e1.record()
    torch.cuda.synchronize()
    print(f"pendulum 4096, body_contacts={int(on)}: {e0.elapsed_time(e1) / (48 * 20):.5f} ms per tick (CUDA-graph replay), "
          f"body-contact mask nonzero on {int((env.sim.get_body_contacts()[:, 0] != 0).sum())} envs")
    env.close()
