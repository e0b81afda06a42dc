#!/usr/bin/env python
"""Cost of the UpkieBaseVelocity tick: the torch epilogue against the fused post-step kernel (developer tool, GPU).

    python tools/base_velocity_cost.py [--rounds 5] [--steps 200] [--warmup 50] [--envs 4096,65536] [--limit 400]

For each batch size, four B200VectorEnv("base_velocity") handles run the same actions:
  torch      the epilogue as a chain of torch launches: base_velocity_tick with the env's CUDA callables (MPC step,
             gyropod step, spine observation), i.e. the tick before k_base_velocity_post existed;
  disabled   step_tensors with autoreset_mode="disabled": the same MPC / step / spine launches, then one
             k_base_velocity_post;
  next_step, same_step   step_tensors with the fused auto-resets and max_episode_steps = --limit, so that envs
             reset during the timed window (same_step includes its one host synchronisation per tick).
The paths alternate ROUNDS times, CUDA events around STEPS ticks after WARMUP. A separate short run under
torch.profiler counts the device kernels and memory operations per tick of each path. The card's name and power
limit are read in the same run. Prints one JSON line per batch size.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

PATHS = ("torch", "disabled", "next_step", "same_step")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--envs", default="4096,65536")
    ap.add_argument("--limit", type=int, default=400)
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile

    from upkie_b200.base_velocity import base_velocity_tick
    from upkie_b200.envs import B200VectorEnv

    if not torch.cuda.is_available():
        raise SystemExit("base_velocity_cost.py needs a CUDA device")
    name = card()
    for n in (int(x) for x in args.envs.split(",")):
        gen = torch.Generator(device="cuda")
        gen.manual_seed(2026)
        acts = [((torch.rand((n, 2), device="cuda", generator=gen) * 2 - 1) * 0.5).contiguous() for _ in range(8)]
        envs = {}
        for p in PATHS:
            mode = "disabled" if p in ("torch", "disabled") else p
            envs[p] = B200VectorEnv(n, "base_velocity", autoreset_mode=mode,
                                    max_episode_steps=0 if mode == "disabled" else args.limit)
            envs[p].reset(seed=3)

        def tick(p, k):
            e = envs[p]
            if p == "torch":
                obs, rew, te, tr, e._spine = base_velocity_tick(acts[k % 8], e._spine, e._xy, e.dt,
                                                                e.mpc_balancer.step_spine, e.sim.step_gyropod,
                                                                e.sim.spine_obs)
                return obs
            return e.step_tensors(acts[k % 8])[0]

        last = {}
        for p in PATHS:
            for k in range(args.warmup):
                last[p] = tick(p, k)
        torch.cuda.synchronize()
        runs = {p: [] for p in PATHS}
        k0 = args.warmup
        for _ in range(args.rounds):
            for p in PATHS:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for k in range(k0, k0 + args.steps):
                    last[p] = tick(p, k)
                e1.record()
                e1.synchronize()
                runs[p].append(e0.elapsed_time(e1) / args.steps)
            k0 += args.steps
        identical = bool(torch.equal(last["torch"], last["disabled"])) and bool(
            torch.equal(envs["torch"].mpc_balancer.commanded_velocity, envs["disabled"].mpc_balancer.commanded_velocity))
        # launches per tick, in a profiled run of its own (not timed)
        launches = {}
        ticks = 20
        for p in PATHS:
            torch.cuda.synchronize()
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for k in range(ticks):
                    tick(p, k0 + k)
                torch.cuda.synchronize()
            dev = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
            mem = sum(1 for e in dev if e.name.startswith(("Memcpy", "Memset")))
            launches[p] = {"kernels": (len(dev) - mem) / ticks, "memory_ops": mem / ticks}
        out = {"card": name, "envs": n, "max_episode_steps": args.limit, "steps_per_round": args.steps,
               "ms_per_tick": {p: {"median": statistics.median(r), "min": min(r), "max": max(r), "runs": r}
                               for p, r in runs.items()},
               "launches_per_tick": launches, "disabled_outputs_identical_to_torch": identical}
        print(json.dumps(out), flush=True)
        for e in envs.values():
            e.close()


if __name__ == "__main__":
    main()
