#!/usr/bin/env python
"""Cost of the servo torque scales per tick (developer tool, needs the GPU).

    python tools/torque_scale_cost.py [--rounds 5] [--steps 400] [--warmup 100] [--out PATH]

Two workloads, both with next-step auto-reset and max_episode_steps = 100, in the observation-delay family (FAM_SENSE,
reached through a servo-dropout spec of probability 0, so that both arms run the same kernels):
  servos     65 536 UpkieServos envs (the headline's physics: fall termination, joint limits, compact rows on device
             buffers),
  pendulum   4 096 UpkiePendulum envs.
Each workload is timed in three arms, with CUDA events around STEPS steps after WARMUP:
  drop0      the zero-probability dropout spec only,
  scale      the same plus torque scales drawn from (0.8, 1.2) on every joint,
  unit       the same with scales of exactly 1 (every statement of the feature runs, the physics is drop0's).
Every round builds fresh handles and runs the arms one after the other, so that they alternate.
Prints one JSON line with ms per tick per workload, arm and round, the medians, the ratios to drop0, and the card's
name, power limit and SM clocks (read in the same run); --out also writes it to a file.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

SCALE = (0.8, 1.2)
WORKLOADS = {"servos": 65536, "pendulum": 4096}


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()

    import torch

    from upkie_b200 import _abi
    from upkie_b200.model import Model
    from upkie_b200.sim import AUTORESET_NEXT_STEP, UpkieSim

    if not torch.cuda.is_available():
        raise SystemExit("torque_scale_cost.py needs a CUDA device")
    model = Model.standard_upkie()
    dev = torch.device("cuda", 0)
    cfg = _abi.default_sim_config()  # bench.py servos_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.max_episode_steps = 100

    gen = torch.Generator(device=dev)
    gen.manual_seed(2025)
    acts = {"servos": [], "pendulum": []}
    tau = torch.tensor(model.tau_max, dtype=torch.float32, device=dev)
    for _ in range(8):
        n = WORKLOADS["servos"]
        a = torch.zeros((n, 6, 6), device=dev)
        a[:, :, 0] = float("nan")
        a[:, :, 5] = tau
        a[:, :, 2] = (torch.rand((n, 6), device=dev, generator=gen) * 2 - 1) * tau
        acts["servos"].append(a.contiguous())
        n = WORKLOADS["pendulum"]
        acts["pendulum"].append(((torch.rand((n, 1), device=dev, generator=gen) * 2 - 1) * 2.0).contiguous())

    def make(workload, arm):
        sim = UpkieSim(WORKLOADS[workload], model=model, config=cfg)
        sim.set_servo_dropout(0.0, 0.0)
        if arm != "drop0":
            sim.set_torque_scale(SCALE if arm == "scale" else (1.0, 1.0))
        sim.set_autoreset(AUTORESET_NEXT_STEP, 2025, 0)
        sim.reset(seed=2025)
        return sim

    def time_arm(workload, arm):
        sim = make(workload, arm)
        step = sim.step_servos_compact if workload == "servos" else sim.step_pendulum
        a = acts[workload]
        for k in range(args.warmup):
            step(a[k % 8])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(args.warmup, args.warmup + args.steps):
            step(a[k % 8])
        e1.record()
        e1.synchronize()
        sim.close()
        return e0.elapsed_time(e1) / args.steps

    runs = {w: {"drop0": [], "scale": [], "unit": []} for w in WORKLOADS}
    for _ in range(args.rounds):
        for w in WORKLOADS:
            for arm in ("drop0", "scale", "unit"):
                runs[w][arm].append(time_arm(w, arm))
    med = {w: {arm: statistics.median(r) for arm, r in arms.items()} for w, arms in runs.items()}
    line = json.dumps({
        "card": card(), "steps_per_round": args.steps, "envs": WORKLOADS, "scale": SCALE,
        "ms_per_tick": {w: {arm: {"median": med[w][arm], "min": min(r), "max": max(r), "runs": r}
                            for arm, r in arms.items()} for w, arms in runs.items()},
        "scale_over_drop0": {w: med[w]["scale"] / med[w]["drop0"] for w in WORKLOADS},
        "unit_over_drop0": {w: med[w]["unit"] / med[w]["drop0"] for w in WORKLOADS},
    })
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
