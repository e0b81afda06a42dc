#!/usr/bin/env python
"""Summarise Nsight Compute outputs into profiles/ (run on the files a profiling run wrote).

    python tools/ncu_summary.py reports/prof_step_r01.ncu-rep reports/launches_r01.csv r01
"""
import collections
import csv
import io
import re
import subprocess
import sys

rep, launches, tag = sys.argv[1], sys.argv[2], sys.argv[3]
# optional: --sidecar servos:limits3:n65536  -> profiles/ncu_sidecar.json[source hash of this build][key], read by bench.py
sidecar_key = sys.argv[sys.argv.index("--sidecar") + 1] if "--sidecar" in sys.argv else None
out = []

# ---- launch list -------------------------------------------------------------------
rows = [r for r in csv.reader(open(launches)) if len(r) > 10 and r[0].isdigit()]
agg = collections.defaultdict(list)
for r in rows:
    name = re.sub(r"\(.*", "", r[4])[:70]
    agg[name].append(float(r[-1]))
total = sum(sum(v) for v in agg.values())
out.append(f"# ncu summary {tag}\n")
out.append("## Launch list of the timed region (`ncu --metrics gpu__time_duration.sum --clock-control none`, "
           "`--profile-from-start off` around bench.py's timed + e2e loops)\n")
out.append("| kernel | launches | total us | avg us | share |\n|---|---:|---:|---:|---:|")
for k, v in sorted(agg.items(), key=lambda kv: -sum(kv[1])):
    out.append(f"| `{k}` | {len(v)} | {sum(v)/1e3:.1f} | {sum(v)/len(v)/1e3:.2f} | {100*sum(v)/total:.1f}% |")

# ---- full-set metrics ------------------------------------------------------------------
raw = subprocess.run(["ncu", "-i", rep, "--page", "raw", "--csv"], capture_output=True, text=True).stdout
rr = list(csv.reader(io.StringIO(raw)))
hdr, units, vals = rr[0], rr[1], rr[2]
d = dict(zip(hdr, vals))
u = dict(zip(hdr, units))
keys = [
    "gpu__time_duration.sum", "launch__grid_size", "launch__block_size", "launch__registers_per_thread",
    "launch__occupancy_limit_registers", "launch__waves_per_multiprocessor",
    "dram__bytes_read.sum", "dram__bytes_write.sum", "gpu__dram_throughput.avg.pct_of_peak_sustained_elapsed",
    "smsp__inst_executed.sum", "smsp__issue_active.avg.pct_of_peak_sustained_active",
    "sm__warps_active.avg.pct_of_peak_sustained_active", "sm__throughput.avg.pct_of_peak_sustained_elapsed",
    "sm__inst_executed_pipe_fma.sum", "sm__inst_executed_pipe_alu.sum", "sm__inst_executed_pipe_fmaheavy.sum",
    "smsp__thread_inst_executed_per_inst_executed.ratio", "l1tex__t_sector_hit_rate.pct", "lts__t_sector_hit_rate.pct",
    "sm__cycles_elapsed.avg", "smsp__cycles_active.avg",
]
out.append(f"\n## `{d.get('Kernel Name', '')[:80]}` (`ncu --set full --clock-control none --import-source on`)\n")
out.append("| metric | value | unit |\n|---|---:|---|")
for k in keys:
    if k in d:
        out.append(f"| {k} | {d[k]} | {u[k]} |")

# ---- SASS opcode mix and stall reasons -----------------------------------------------------
src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
sr = list(csv.reader(io.StringIO(src)))
h2 = sr[1]
iS, iE = h2.index("Source"), h2.index("Instructions Executed")
stall_cols = [(i, h) for i, h in enumerate(h2) if h.startswith("stall_") and "Not Issued" not in h]
ops, stalls, tot, static = collections.Counter(), collections.Counter(), 0, 0
for r in sr[2:]:
    if len(r) < len(h2):
        if r and r[0] == "Kernel Name":
            break
        continue
    try:
        e = int(r[iE])
    except ValueError:
        continue
    static += 1
    m = re.match(r"\s*(@!?U?P\d+\s+)?([A-Z0-9_.]+)", r[iS])
    ops[m.group(2).split(".")[0] if m else "?"] += e
    tot += e
    for i, h in stall_cols:
        try:
            stalls[h] += int(r[i])
        except ValueError:
            pass
warps = int(float(d.get("launch__grid_size", "1"))) * int(float(d.get("launch__block_size", "32"))) // 32
out.append(f"\nStatic SASS instructions: {static} ({static * 16 / 1024:.0f} KB). Dynamic warp instructions: {tot} "
           f"= {tot / max(1, warps):.0f} per warp (= per env-step).\n")
out.append("| opcode | share | per env-step |\n|---|---:|---:|")
for op, c in ops.most_common(14):
    out.append(f"| {op} | {100*c/tot:.2f}% | {c/max(1, warps):.0f} |")
st = sum(stalls.values())
out.append("\n| warp stall reason (sampled) | share |\n|---|---:|")
for h, c in stalls.most_common(8):
    out.append(f"| {h} | {100*c/st:.1f}% |")
print("\n".join(out))

if sidecar_key:
    import json
    import os

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path.insert(0, root)
    from upkie_b200 import build as b

    def num(key):
        v = float(d[key].replace(",", ""))
        unit = u[key].lower()
        return v * {"byte": 1, "kbyte": 1e3, "mbyte": 1e6, "gbyte": 1e9}.get(unit, 1)

    fp_ops = ("FFMA2", "FMUL2", "FADD2", "FFMA", "FMUL", "FADD")
    entry = {
        "kernel": d.get("Kernel Name", "")[:60],
        "dram_bytes": int(num("dram__bytes_read.sum") + num("dram__bytes_write.sum")),
        "instr_per_env_step": tot / max(1, warps),
        "fp_instr_share": sum(ops[o] for o in fp_ops) / max(1, tot),
        "issue_active_pct": float(d["smsp__issue_active.avg.pct_of_peak_sustained_active"]),
        "duration_us_under_ncu": float(d["gpu__time_duration.sum"]),
        "report": os.path.basename(rep),
        "captured": "one launch, `ncu --set full --clock-control none`, steady state (launch 200 of the bench loop)",
    }
    path = os.path.join(root, "profiles", "ncu_sidecar.json")
    data = json.load(open(path)) if os.path.exists(path) else {}
    data.setdefault(b.source_hash(), {})[sidecar_key] = entry
    with open(path, "w") as f:
        json.dump(data, f, indent=1)
    print(f"\nsidecar: profiles/ncu_sidecar.json[{b.source_hash()}][{sidecar_key}] = {entry}", file=sys.stderr)
