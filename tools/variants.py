#!/usr/bin/env python
"""Build-time variant explorer for the step kernel (developer tool).

    python tools/variants.py build      # here (no GPU): compiles variants/lib_<name>.so
    python tools/variants.py run [names]  # on the GPU box: times each variant with bench.py (UPKIE_B200_LIB)

Round 2: the variants differ in the translation unit of the benchmarked kernel only (step_host_limits.cu: TILE=1,
extras + joint-limit rows); every other object is taken from the in-tree build (upkie_b200/build/*.o).
"""
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
CSRC = os.path.join(ROOT, "upkie_b200", "csrc")
OBJ = os.path.join(ROOT, "upkie_b200", "build")
OUT = os.path.join(ROOT, "variants")
VARIANTS = {
    "new_paired": [],
    "new_scalarW": ["-DUPKIE_TENROW_PAIRED_COLS=0"],
    "v1": ["-DUPKIE_TENROW_V1=1"],
}
UNIT = "step_host_limits"
KERNEL = "k_stepILi0ELi1ELi2ELi1E"


def build():
    from upkie_b200 import build as b

    b.build()
    os.makedirs(OUT, exist_ok=True)
    procs = []
    for name, flags in VARIANTS.items():
        obj = os.path.join(OUT, f"{UNIT}_{name}.o")
        cmd = ["nvcc"] + b.NVCC_FLAGS + flags + ["-Xptxas", "-v", "-c", "-o", obj, os.path.join(CSRC, UNIT + ".cu")]
        procs.append((name, obj, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)))
    for name, obj, p in procs:
        out, _ = p.communicate()
        lines = out.splitlines()
        info = ""
        for i, l in enumerate(lines):
            if KERNEL in l and "Function properties" in l:
                info = " | ".join(x.strip() for x in lines[i + 1:i + 3])
        objs = [os.path.join(OBJ, os.path.splitext(s)[0] + ".o") for s in b.SOURCES if not s.startswith(UNIT)] + [obj]
        rc = subprocess.call(["nvcc"] + b.GENCODE + ["-shared", "-o", os.path.join(OUT, f"lib_{name}.so")] + objs)
        print(f"{name:16s} rc={p.returncode}/{rc} {info}")


def run():
    names = sys.argv[2:] or list(VARIANTS)
    for name in names:
        try:
            env = dict(os.environ, UPKIE_B200_LIB=os.path.join(OUT, f"lib_{name}.so"))
            r = subprocess.run([sys.executable, os.path.join(ROOT, "bench.py"), "--steps", "300", "--warmup", "20",
                                "--no-cpu-baseline", "--no-other-workloads"], env=env, capture_output=True, text=True, timeout=200)
            try:
                j = json.loads(r.stdout.strip().splitlines()[-1])
                print(f"{name:16s} value={j['value']:.4e} kernel_ms={j['roofline']['kernel_ms']:.4f} "
                      f"ms_per_step={j['ms_per_step']:.4f} e2e={j['e2e']['value']:.3e}", flush=True)
            except Exception:
                print(name, "FAILED", r.stdout[-300:], r.stderr[-600:], flush=True)
        except subprocess.TimeoutExpired:
            print(name, "TIMEOUT", flush=True)


if __name__ == "__main__":
    {"build": build, "run": run}[sys.argv[1]]()
