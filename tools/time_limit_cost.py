#!/usr/bin/env python
"""Cost of the episode time limit on the headline workload (developer tool, needs the GPU).

    python tools/time_limit_cost.py [--rounds 5] [--steps 400] [--warmup 100] [--limit 1000]

65 536 UpkieServos envs, the headline's physics (BASELINE configs[2]: fall termination, joint limits, random
torques, randomised friction and inertias), next-step auto-reset, compact rows on device buffers: the kernel of
bench.py's headline. It times the step with the limit off (`step_servos_compact`, what bench.py runs) and with
`max_episode_steps = --limit` (`upkie_b200_step` with compact rows and `truncated`), alternating the two handles
ROUNDS times, with CUDA events around STEPS steps after WARMUP. Prints one JSON line with ms per tick per round,
the medians, and the card's name and power limit.
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
    ap.add_argument("--limit", type=int, default=1000)
    ap.add_argument("--envs", type=int, default=65536)
    args = ap.parse_args()

    import torch

    from upkie_b200 import _abi
    from upkie_b200.model import Model
    from upkie_b200.sim import AUTORESET_NEXT_STEP, UpkieSim

    if not torch.cuda.is_available():
        raise SystemExit("time_limit_cost.py needs a CUDA device")
    model = Model.standard_upkie()
    n = args.envs
    dev = torch.device("cuda", 0)
    gen = torch.Generator(device=dev)
    gen.manual_seed(2025)
    mu = torch.empty(n, device=dev).uniform_(0.5, 1.2, generator=gen)
    eps = torch.empty((n, 6), device=dev).uniform_(-0.2, 0.2, generator=gen)
    tau = torch.tensor(model.tau_max, dtype=torch.float32, device=dev)
    acts = []
    for _ in range(8):
        a = torch.zeros((n, 6, 6), device=dev)
        a[:, :, 0] = float("nan")
        a[:, :, 5] = tau
        a[:, :, 2] = (torch.rand((n, 6), device=dev, generator=gen) * 2 - 1) * tau
        acts.append(a.contiguous())

    def make(limit):
        cfg = _abi.default_sim_config()  # bench.py servos_config()
        cfg.servos_fall_termination = 1
        cfg.min_base_height = 0.15
        cfg.rand_pitch = 0.3
        cfg.max_episode_steps = limit
        sim = UpkieSim(n, model=model, config=cfg)
        sim.set_randomization(friction=mu, inertia_eps=eps)
        sim.set_autoreset(AUTORESET_NEXT_STEP, 2025, 0)
        sim.reset(seed=2025)
        return sim

    sims = {"off": make(0), "on": make(args.limit)}
    step = {"off": lambda k: sims["off"].step_servos_compact(acts[k % 8]),
            "on": lambda k: sims["on"].step_servos_compact_truncated(acts[k % 8])}
    for name in sims:
        for k in range(args.warmup):
            step[name](k)
    torch.cuda.synchronize()
    runs = {name: [] for name in sims}
    k0 = args.warmup
    for _ in range(args.rounds):
        for name in sims:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(k0, k0 + args.steps):
                step[name](k)
            e1.record()
            e1.synchronize()
            runs[name].append(e0.elapsed_time(e1) / args.steps)
        k0 += args.steps
    out ={"card": card(), "envs": n, "max_episode_steps": args.limit, "steps_per_round": args.steps,
           "ms_per_tick": {name: {"median": statistics.median(r), "min": min(r), "max": max(r), "runs": r}
                           for name, r in runs.items()}}
    out["on_over_off"] = out["ms_per_tick"]["on"]["median"] / out["ms_per_tick"]["off"]["median"]
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
