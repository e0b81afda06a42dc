#!/usr/bin/env python
"""Cost of the spine-rate observation history per tick (developer tool, needs the GPU).

    python tools/history_cost.py [--rounds 5] [--steps 400] [--warmup 100]

Two workloads: 65 536 UpkieServos envs (the headline's physics: fall termination, joint limits, compact rows on
device buffers) and 4 096 UpkiePendulum envs, both with next-step auto-reset and max_episode_steps = 100. Each times
three handles, alternating them ROUNDS times, with CUDA events around STEPS steps after WARMUP:
  sense0   a parameter table equal to the config's values and an observation delay of 0 substeps (FAM_SENSE),
  k5c4     that handle plus a history of K = 5 entries of C = 4 columns (one tick of pitch and the IMU rates),
  k40c16   that handle plus a history of K = 40 entries of C = 16 columns (both IMU accelerations among them).
Prints one JSON line with ms per tick per round, the medians, and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=100)
    args = ap.parse_args()

    import torch

    from upkie_b200 import _abi
    from upkie_b200.model import Model
    from upkie_b200.sim import AUTORESET_NEXT_STEP, UpkieSim

    if not torch.cuda.is_available():
        raise SystemExit("history_cost.py needs a CUDA device")
    model = Model.standard_upkie()
    dev = torch.device("cuda", 0)
    cfg = _abi.default_sim_config()  # bench.py servos_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.max_episode_steps = 100
    A = _abi
    small = [A.SP_PITCH] + list(range(A.SP_IMU_ANGVEL, A.SP_IMU_ANGVEL + 3))
    large = (list(range(A.SP_BASE_ANGVEL, A.SP_BASE_ANGVEL + 3)) + [A.SP_PITCH]
             + list(range(A.SP_IMU_ANGVEL, A.SP_IMU_RAWACC + 3)) + [A.SP_SERVO + 2 * 5 + 1, A.SP_SERVO + 5 * 5 + 1,
                                                                  A.SP_SERVO + 2 * 5 + 2])
    assert len(small) == 4 and len(large) == 16
    HISTORIES = {"k5c4": (small, 5), "k40c16": (large, 40)}

    def actions(kind, n, gen):
        out = []
        for _ in range(8):
            if kind == "servos":
                tau = torch.tensor(model.tau_max, dtype=torch.float32, device=dev)
                a = torch.zeros((n, 6, 6), device=dev)
                a[:, :, 0] = float("nan")
                a[:, :, 5] = tau
                a[:, :, 2] = (torch.rand((n, 6), device=dev, generator=gen) * 2 - 1) * tau
            else:
                a = (torch.rand((n, 1), device=dev, generator=gen) * 2 - 1) * 2.0
            out.append(a.contiguous())
        return out

    def make(n, arm):
        sim = UpkieSim(n, model=model, config=cfg)
        rows = torch.from_numpy(_abi.config_env_params(cfg)).to(dev).expand(n, _abi.EP_DIM).contiguous()
        sim.set_env_params(rows)
        sim.set_observation_delay(0, 0)
        if arm in HISTORIES:
            sim.set_history(*HISTORIES[arm])
        sim.set_autoreset(AUTORESET_NEXT_STEP, 2025, 0)
        sim.reset(seed=2025)
        sim.obs_servos_compact = torch.empty((n, 6, 3), dtype=torch.float32, device=dev)  # one output per handle
        return sim

    result = {"card": card(), "steps_per_round": args.steps}
    for kind, n in (("servos", 65536), ("pendulum", 4096)):
        gen = torch.Generator(device=dev)
        gen.manual_seed(2025)
        acts = actions(kind, n, gen)
        sims = {arm: make(n, arm) for arm in ("sense0", "k5c4", "k40c16")}

        def step(sim, k):
            if kind == "servos":
                sim.step_servos_compact(acts[k % 8])
            else:
                sim.step_pendulum(acts[k % 8])

        for sim in sims.values():
            for k in range(args.warmup):
                step(sim, k)
        torch.cuda.synchronize()
        runs = {arm: [] for arm in sims}
        k0 = args.warmup
        for _ in range(args.rounds):
            for arm, sim in sims.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for k in range(k0, k0 + args.steps):
                    step(sim, k)
                e1.record()
                e1.synchronize()
                runs[arm].append(e0.elapsed_time(e1) / args.steps)
            k0 += args.steps
        med = {arm: statistics.median(r) for arm, r in runs.items()}
        result[kind] = {
            "envs": n,
            "ms_per_tick": {arm: {"median": med[arm], "min": min(r), "max": max(r), "runs": r} for arm, r in runs.items()},
            "k5c4_over_sense0": med["k5c4"] / med["sense0"],
            "k40c16_over_sense0": med["k40c16"] / med["sense0"],
        }
        for sim in sims.values():
            sim.close()
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
