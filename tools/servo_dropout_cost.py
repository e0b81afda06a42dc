#!/usr/bin/env python
"""Cost of the servo reply dropouts per tick (developer tool, needs the GPU).

    python tools/servo_dropout_cost.py [--rounds 5] [--steps 400] [--warmup 100] [--tree NAME=DIR ...]

65 536 UpkieServos envs (the headline's physics: fall termination, joint limits, compact rows on device buffers) with
next-step auto-reset and max_episode_steps = 100. Times handles of the observation-delay family (FAM_SENSE: a parameter
table equal to the config's values and an observation delay of 0 substeps), with CUDA events around STEPS steps after
WARMUP:
  sense0   no dropouts,
  p0       dropouts of every servo with probability 0 (the branch runs, nothing is lost),
  p05      dropouts of every servo with probabilities drawn from U(0, 0.1) at each reset.
Each `--tree NAME=DIR` adds another build to compare: DIR holds an `upkie_b200` package with its built library (another
revision of the kernels). Every round then runs each build in a process of its own, one after the other, so that the
builds alternate; a build whose package has no servo dropouts times sense0 only.
Prints one JSON line with ms per tick per build, arm and round, the medians, and the card's name and power limit.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def measure(args):
    """one round of every arm the package on sys.path has, ms per tick"""
    import torch

    from upkie_b200 import _abi
    from upkie_b200.model import Model
    from upkie_b200.sim import AUTORESET_NEXT_STEP, UpkieSim

    if not torch.cuda.is_available():
        raise SystemExit("servo_dropout_cost.py needs a CUDA device")
    model = Model.standard_upkie()
    dev = torch.device("cuda", 0)
    cfg = _abi.default_sim_config()  # bench.py servos_config()
    cfg.servos_fall_termination = 1
    cfg.min_base_height = 0.15
    cfg.rand_pitch = 0.3
    cfg.max_episode_steps = 100
    dropouts = {"p0": (0.0, 0.0), "p05": (0.0, 0.1)} if hasattr(UpkieSim, "set_servo_dropout") else {}
    n = 65536

    gen = torch.Generator(device=dev)
    gen.manual_seed(2025)
    acts = []
    for _ in range(8):
        tau = torch.tensor(model.tau_max, dtype=torch.float32, device=dev)
        a = torch.zeros((n, 6, 6), device=dev)
        a[:, :, 0] = float("nan")
        a[:, :, 5] = tau
        a[:, :, 2] = (torch.rand((n, 6), device=dev, generator=gen) * 2 - 1) * tau
        acts.append(a.contiguous())

    def make(arm):
        sim = UpkieSim(n, model=model, config=cfg)
        rows = torch.from_numpy(_abi.config_env_params(cfg)).to(dev).expand(n, _abi.EP_DIM).contiguous()
        sim.set_env_params(rows)
        sim.set_observation_delay(0, 0)
        if arm in dropouts:
            sim.set_servo_dropout(*dropouts[arm])
        sim.set_autoreset(AUTORESET_NEXT_STEP, 2025, 0)
        sim.reset(seed=2025)
        return sim

    out = {}
    for arm in ["sense0"] + list(dropouts):
        sim = make(arm)
        for k in range(args.warmup):
            sim.step_servos_compact(acts[k % 8])
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for k in range(args.warmup, args.warmup + args.steps):
            sim.step_servos_compact(acts[k % 8])
        e1.record()
        e1.synchronize()
        out[arm] = e0.elapsed_time(e1) / args.steps
        sim.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=400)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--tree", action="append", default=[], help="NAME=DIR: another build to alternate with")
    ap.add_argument("--child", action="store_true", help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:  # one round of the package first on sys.path (PYTHONPATH)
        print(json.dumps(measure(args)), flush=True)
        return
    trees = {"this": ROOT}
    for t in args.tree:
        name, _, path = t.partition("=")
        trees[name] = os.path.abspath(path)
    runs = {name: {} for name in trees}
    for _ in range(args.rounds):
        for name, path in trees.items():
            env = dict(os.environ, PYTHONPATH=path)
            env.pop("UPKIE_B200_LIB", None)
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", "--steps", str(args.steps),
                                "--warmup", str(args.warmup)], env=env, cwd=path, capture_output=True, text=True)
            if r.returncode != 0:
                raise SystemExit(f"{name}: {r.stderr[-2000:]}")
            for arm, ms in json.loads(r.stdout.strip().splitlines()[-1]).items():
                runs[name].setdefault(arm, []).append(ms)
    med = {name: {arm: statistics.median(r) for arm, r in arms.items()} for name, arms in runs.items()}
    result = {
        "card": card(), "steps_per_round": args.steps, "envs": 65536,
        "ms_per_tick": {name: {arm: {"median": med[name][arm], "min": min(r), "max": max(r), "runs": r}
                               for arm, r in arms.items()} for name, arms in runs.items()},
        "over_sense0": {name: {arm: m / med[name]["sense0"] for arm, m in arms.items() if arm != "sense0"}
                        for name, arms in med.items()},
    }
    if len(trees) > 1:
        result["sense0_over_this"] = {name: med[name]["sense0"] / med["this"]["sense0"] for name in trees}
    print(json.dumps(result), flush=True)


if __name__ == "__main__":
    main()
