#!/usr/bin/env python
"""Before / after comparison of the step kernel library (developer tool).

    python tools/ab_step.py build [REV]   # no GPU needed: extracts REV (default HEAD) into build/ab_step/base,
                                          # builds its libraries there, and builds the working tree's
    python tools/ab_step.py run [OUT]     # on the GPU: times both revisions with bench.py, alternating, and
                                          # compares their outputs; writes OUT (default build/ab_step/out)

`run` times each revision with its own checkout: the old one runs build/ab_step/base/bench.py with its own Python
package and libraries (cwd build/ab_step/base), the new one the working tree's. So the two may differ in their C ABI
(include/upkie_b200.h). It runs, in this order:
  - bench.py --no-cpu-baseline --no-other-workloads, old / new alternating, ROUNDS times each (the headline);
  - bench.py --no-cpu-baseline --dump-outputs once per revision (same seeds): obs / terminated compared with
    numpy.array_equal, and the secondary workloads of that run (exact mode: each revision's own exact library);
and prints one JSON summary line with the card's name and power limit.
"""
import json
import os
import shutil
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BASE = os.path.join(ROOT, "build", "ab_step", "base")
TREES = {"old": BASE, "new": ROOT}
LIBS = {name: os.path.join(tree, "upkie_b200", "libupkie_b200.so") for name, tree in TREES.items()}
ROUNDS = 5


def build():
    rev = sys.argv[2] if len(sys.argv) > 2 else "HEAD"
    shutil.rmtree(BASE, ignore_errors=True)
    os.makedirs(BASE)
    archive = subprocess.run(["git", "-C", ROOT, "archive", rev], check=True, capture_output=True).stdout
    subprocess.run(["tar", "-x", "-C", BASE], input=archive, check=True)
    build_lib = ("import sys; sys.path.insert(0, '.'); from upkie_b200 import build; "
                 "print(build.build(force=True), build.build_exact(force=True))")
    procs = [subprocess.Popen([sys.executable, "-c", build_lib], cwd=d) for d in (BASE, ROOT)]
    if any(p.wait() for p in procs):
        raise SystemExit("ab_step: library build failed")
    with open(os.path.join(BASE, "REV"), "w") as f:
        f.write(subprocess.run(["git", "-C", ROOT, "rev-parse", rev], check=True, capture_output=True,
                               text=True).stdout)


def bench(tree, extra):
    env = {k: v for k, v in os.environ.items() if k != "UPKIE_B200_LIB"}
    r = subprocess.run([sys.executable, os.path.join(tree, "bench.py"), "--gpus", "1", "--no-cpu-baseline"] + extra,
                       env=env, capture_output=True, text=True, cwd=tree)
    if r.returncode != 0:
        raise SystemExit(f"bench.py failed in {tree}:\n{r.stdout[-2000:]}\n{r.stderr[-4000:]}")
    return json.loads(r.stdout.strip().splitlines()[-1])


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True).stdout.strip().splitlines()
    return q[0] if q else "unknown"


def run():
    import numpy as np

    # absolute: the old revision's bench.py runs with its own checkout as working directory
    out = os.path.abspath(sys.argv[2] if len(sys.argv) > 2 else os.path.join(ROOT, "build", "ab_step", "out"))
    os.makedirs(out, exist_ok=True)
    for name, lib in LIBS.items():
        if not os.path.exists(lib):
            raise SystemExit(f"ab_step: {lib} missing; run `python tools/ab_step.py build` first")
    rev_file = os.path.join(BASE, "REV")
    summary = {"card": card(), "base_rev": open(rev_file).read().strip() if os.path.exists(rev_file) else None}
    head = {name: [] for name in LIBS}
    for _ in range(ROUNDS):
        for name, tree in TREES.items():
            j = bench(tree, ["--no-other-workloads"])
            head[name].append({"ms_per_step": j["ms_per_step"], "kernel_ms": j["roofline"]["kernel_ms"],
                               "sm_mhz": j["clocks"].get("sm_mhz"), "power_limit_w": j["clocks"].get("power_limit_w")})
            print(name, json.dumps(head[name][-1]), flush=True)
    summary["headline"] = {}
    for name, runs in head.items():
        ms = [r["ms_per_step"] for r in runs]
        summary["headline"][name] = {"ms_per_step_median": statistics.median(ms), "min": min(ms), "max": max(ms),
                                     "kernel_ms_median": statistics.median(r["kernel_ms"] for r in runs), "runs": runs}
    old_ms = summary["headline"]["old"]["ms_per_step_median"]
    summary["headline"]["speedup"] = old_ms / summary["headline"]["new"]["ms_per_step_median"]
    full = {}
    for name, tree in TREES.items():
        j = bench(tree, ["--dump-outputs", os.path.join(out, name)])
        full[name] = j
        with open(os.path.join(out, f"bench_{name}.json"), "w") as f:
            json.dump(j, f)
    summary["other_workloads"] = {
        w: {name: full[name]["other_workloads"][w].get("ms_per_step") for name in LIBS}
        for w in full["new"].get("other_workloads", {})}
    same = {}
    for fn in sorted(os.listdir(os.path.join(out, "new"))):
        a, b = np.load(os.path.join(out, "old", fn)), np.load(os.path.join(out, "new", fn))
        same[fn] = bool(np.array_equal(a, b, equal_nan=a.dtype.kind == "f"))
    summary["outputs_bit_identical"] = same
    with open(os.path.join(out, "summary.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps({k: v for k, v in summary.items() if k != "headline"} | {
        "headline": {k: (v if k == "speedup" else {kk: vv for kk, vv in v.items() if kk != "runs"})
                     for k, v in summary["headline"].items()}}), flush=True)


if __name__ == "__main__":
    {"build": build, "run": run}[sys.argv[1]]()
