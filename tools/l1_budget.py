#!/usr/bin/env python
# SPDX-License-Identifier: Apache-2.0
"""Headline tick time against the L1 the step kernel's local-memory frame can use (developer tool, needs a GPU).

    python tools/l1_budget.py [ROUNDS]     # default 5 rounds

An SM of the H100 splits 256 KB between shared memory (the carveout: 0, 8, 16, 32, 64, 100, 132, 164, 196 or 228 KB)
and L1, where the headline kernel's spill frame (bytes per thread x 256 threads per block) lives when it hits. Each
setting runs `bench.py --no-cpu-baseline --no-other-workloads` in a process of its own with
UPKIE_STEP_SMEM_CARVEOUT set (read when the handle is created): -1 leaves the carveout to the driver, 0 is the
library's default (cudaSharedmemCarveoutMaxL1: the smallest carveout that holds the block), the others are the
percentages of 228 KB that round up to 100, 132, 164 and 228 KB. The settings alternate within each round. Prints one
line per setting (ms per tick, median and range) and the card's name, power limit and SM clock.
"""
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
# (label, UPKIE_STEP_SMEM_CARVEOUT): the driver rounds a percentage of 228 KB up to the next carveout step
SETTINGS = [("driver default", -1), ("library default (max L1)", 0), ("100 KB", 43), ("132 KB", 57),
            ("164 KB", 71), ("228 KB", 100)]


def bench(carveout):
    env = dict(os.environ, UPKIE_STEP_SMEM_CARVEOUT=str(carveout))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--gpus", "1", "--no-cpu-baseline",
                        "--no-other-workloads"], env=env, capture_output=True, text=True, cwd=ROOT)
    if r.returncode != 0:
        raise SystemExit(f"bench.py failed (carveout {carveout}):\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def main():
    rounds = int(sys.argv[1]) if len(sys.argv) > 1 else 5
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()
    runs = {label: [] for label, _ in SETTINGS}
    clocks = []
    for _ in range(rounds):
        for label, carveout in SETTINGS:
            j = bench(carveout)
            runs[label].append(j["ms_per_step"])
            clocks.append(j["clocks"].get("sm_mhz"))
            print(json.dumps({"setting": label, "carveout": carveout, "ms_per_step": j["ms_per_step"]}), flush=True)
    print(f"card: {card[0] if card else 'unknown'}; SM clock during the runs (MHz): {sorted(set(clocks))}")
    for label, carveout in SETTINGS:
        ms = runs[label]
        print(f"{label:26s} ({carveout:3d}): {statistics.median(ms):.4f} ms per tick "
              f"(range {min(ms):.4f}-{max(ms):.4f}, {len(ms)} runs)")


if __name__ == "__main__":
    main()
