#!/usr/bin/env python
"""Cost of info["final_info"] (the terminal spine observation of same-step auto-resets) on the headline workload
(developer tool, needs the GPU).

    python tools/final_info_cost.py [--rounds 5] [--steps 400] [--warmup 100] [--limit 100] [--envs 4096,65536]

UpkieServos envs with the headline's physics (bench.py servos_config: fall termination, joint limits, random torques,
randomised friction and inertias), same-step auto-reset and `max_episode_steps = --limit`, so that envs reset on
every tick. Compact rows and `truncated` on device buffers (`upkie_b200_step`). Three variants, one handle each,
alternated ROUNDS times with CUDA events around STEPS steps after WARMUP:
  off    the same-step step without the stash (UpkieStepOutputs.final_state = 0)
  on     the step with final_state = 1: the resetting envs stash their pre-reset state
  fetch  the step with final_state = 1, then `upkie_b200_final_spine_obs` into a device buffer every tick
Prints one JSON line per env count with ms per tick per round, the medians, the kernels per tick (counted with
torch.profiler over a few ticks in a separate pass), the resets per tick (counted at the last tick of each round), and the card's name and power limit.
"""
import argparse
import json
import os
import re
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def measure(n, args, torch, model):
    from upkie_b200 import _abi
    from upkie_b200.sim import AUTORESET_SAME_STEP, UpkieSim

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

    def make():
        cfg = _abi.default_sim_config()  # bench.py servos_config()
        cfg.servos_fall_termination = 1
        cfg.min_base_height = 0.15
        cfg.rand_pitch = 0.3
        cfg.max_episode_steps = args.limit
        sim = UpkieSim(n, model=model, config=cfg)
        sim.set_randomization(friction=mu, inertia_eps=eps)
        sim.set_autoreset(AUTORESET_SAME_STEP, 2025, 0)
        sim.reset(seed=2025)
        return sim

    names = ("off", "on", "fetch")
    sims = {name: make() for name in names}
    rows = torch.zeros((n, _abi.SPINE_DIM), dtype=torch.float32, device=dev)

    def step(name, k):
        s = sims[name]
        s.step_servos_compact_truncated(acts[k % 8], final_state=name != "off")
        if name == "fetch":
            s.final_spine_obs(rows)

    for name in names:
        for k in range(args.warmup):
            step(name, k)
    torch.cuda.synchronize()
    runs = {name: [] for name in names}
    k0 = args.warmup
    resets = 0
    for _ in range(args.rounds):
        for name in names:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(k0, k0 + args.steps):
                step(name, k)
            e1.record()
            e1.synchronize()
            runs[name].append(e0.elapsed_time(e1) / args.steps)
        s = sims["off"]
        resets += int((s.terminated | s.truncated).sum())
        k0 += args.steps

    # kernels per tick, in a pass of its own (tracing slows the host)
    from torch.profiler import ProfilerActivity, profile

    kernels = {}
    ticks = 10
    for name in names:
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for k in range(k0, k0 + ticks):
                step(name, k)
            torch.cuda.synchronize()
        evs = [e for e in prof.events() if e.device_type.name == "CUDA" and "memcpy" not in e.name.lower()
               and "memset" not in e.name.lower()]
        kernels[name] = {"per_tick": len(evs) / ticks,
                         "names": sorted({(re.findall(r"\bk_\w+", e.name) or [e.name])[0] for e in evs})}
    for s in sims.values():
        s.close()
    ms = {name: {"median": statistics.median(r), "min": min(r), "max": max(r), "runs": r} for name, r in runs.items()}
    return {"card": card(), "envs": n, "max_episode_steps": args.limit, "steps_per_round": args.steps,
            "resets_per_tick": resets / args.rounds, "ms_per_tick": ms, "kernels": kernels,
            "on_over_off": ms["on"]["median"] / ms["off"]["median"],
            "fetch_over_off": ms["fetch"]["median"] / ms["off"]["median"]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--limit", type=int, default=100)
    ap.add_argument("--envs", default="4096,65536")
    args = ap.parse_args()

    import torch

    from upkie_b200.model import Model

    if not torch.cuda.is_available():
        raise SystemExit("final_info_cost.py needs a CUDA device")
    model = Model.standard_upkie()
    for n in (int(x) for x in args.envs.split(",")):
        print(json.dumps(measure(n, args, torch, model)), flush=True)


if __name__ == "__main__":
    main()
