#!/usr/bin/env python
"""Cost of reset randomisation on the headline workload (developer tool, needs the GPU).

    python tools/reset_randomization_cost.py [--rounds 5] [--steps 400] [--warmup 100]

65 536 UpkieServos envs, the headline's physics (BASELINE configs[2]: fall termination, joint limits, random
torques, randomised friction and inertias), next-step auto-reset with max_episode_steps = 100, so that about 1 % of
the envs reset per tick, compact rows on device buffers. It times three handles, alternating them ROUNDS times, with
CUDA events around STEPS steps after WARMUP: a parameter table equal to the config's values, reset randomisation with
no column selected, and reset randomisation of all 35 columns (gains, joint friction, torque noise, IMU uncertainty,
inertias, floor friction). The first two handles step the same actions from the same state: the tool checks that
their observations, `terminated` and state stay bit-identical. Prints one JSON line with ms per tick per round, the
medians, the mean share of envs reset per tick, and the card's name and power limit.
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
    ap.add_argument("--envs", type=int, default=65536)
    args = ap.parse_args()

    import torch

    from upkie_b200 import _abi
    from upkie_b200.model import Model
    from upkie_b200.sim import AUTORESET_NEXT_STEP, UpkieSim

    if not torch.cuda.is_available():
        raise SystemExit("reset_randomization_cost.py needs a CUDA device")
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

    cfg = _abi.default_sim_config()  # bench.py servos_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.max_episode_steps = 100
    config_rows = torch.from_numpy(_abi.config_env_params(cfg)).to(dev).expand(n, _abi.EP_DIM).contiguous()
    ranges = ([(15.0, 25.0), (0.5, 1.5)] + [(0.0, 0.05)] * 18 + [(-0.1, 0.1)] * 3 + [(0.0, 0.05)]
              + [(-0.01, 0.01)] * 3 + [(0.0, 0.01)] + [(-0.2, 0.2)] * 6 + [(0.5, 1.2)])

    def spec(columns):
        s = _abi.UpkieResetRandomization()
        s.columns = columns
        for k, (lo, hi) in enumerate(ranges):
            s.low[k], s.high[k] = lo, hi
        return s

    def make(columns):
        sim = UpkieSim(n, model=model, config=cfg)
        sim.set_randomization(friction=mu, inertia_eps=eps)
        sim.set_env_params(config_rows)
        sim.set_autoreset(AUTORESET_NEXT_STEP, 2025, 0)
        sim.reset(seed=2025)
        if columns is not None:
            sim.set_reset_randomization(spec(columns))
        sim.obs_servos_compact = torch.empty((n, 6, 3), dtype=torch.float32, device=dev)  # one output per handle
        return sim

    sims = {"table": make(None), "none_selected": make(0), "all_selected": make((1 << _abi.RR_DIM) - 1)}
    outs = {}

    def step(name, k):
        outs[name] = sims[name].step_servos_compact(acts[k % 8])

    identical = True

    def compare():
        a, b = outs["table"], outs["none_selected"]
        same = all(torch.equal(x, y) for x, y in zip(a, b))
        return same and torch.equal(sims["table"].get_state(), sims["none_selected"].get_state())

    for name in sims:
        for k in range(args.warmup):
            step(name, k)
    torch.cuda.synchronize()
    identical &= compare()
    runs = {name: [] for name in sims}
    k0 = args.warmup
    for _ in range(args.rounds):
        for name in sims:
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for k in range(k0, k0 + args.steps):
                step(name, k)
            e1.record()
            e1.synchronize()
            runs[name].append(e0.elapsed_time(e1) / args.steps)
        identical &= compare()
        k0 += args.steps
    out = {"card": card(), "envs": n, "steps_per_round": args.steps,
           "ms_per_tick": {name: {"median": statistics.median(r), "min": min(r), "max": max(r), "runs": r}
                           for name, r in runs.items()},
           "none_selected_bit_identical": bool(identical)}
    base = out["ms_per_tick"]["table"]["median"]
    out["none_selected_over_table"] = out["ms_per_tick"]["none_selected"]["median"] / base
    out["all_selected_over_table"] = out["ms_per_tick"]["all_selected"]["median"] / base
    draws = sims["all_selected"].get_draws().double().sum().item()
    out["resets_per_env_tick"] = draws / (n * k0)  # draws since the spec was set, one per reset
    print(json.dumps(out), flush=True)
    if not identical:
        raise SystemExit("reset randomisation with no column selected changed the outputs")


if __name__ == "__main__":
    main()
