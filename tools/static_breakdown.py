#!/usr/bin/env python3
# SPDX-License-Identifier: Apache-2.0
"""Static SASS instruction counts of one step kernel, bucketed by the source function each instruction's line
belongs to (needs the library built with -lineinfo, which build.py does). Developer tool, runs without a GPU:

    python tools/static_breakdown.py [kernel-substring]      # default: k_stepILi0ELi1ELi2ELi1E (bench kernel)
    python tools/static_breakdown.py [kernel-substring] --ncu reports/prof.ncu-rep
        # adds DYNAMIC columns from an `ncu --set full --import-source on` capture of the SAME build: warp
        # instructions executed and sampled stall reasons per bucket (joined by instruction index)
    python tools/static_breakdown.py [kernel-substring] --lib build/ab_step/base/upkie_b200/libupkie_b200.so
        # another build of the library, e.g. the base revision that tools/ab_step.py builds

The "substep:" buckets (and `servo_substep`) are inside the `nb_substeps` loop; the PGS bucket holds two inlined
copies of the six-row sweep, each run once per pair of sweeps.
"""
import collections
import os
import re
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LIB = os.path.join(ROOT, "upkie_b200", "libupkie_b200.so")
CSRC = os.path.join(ROOT, "upkie_b200", "csrc")


def function_starts(path):
    """[(line, name)] of function definitions / named lambdas in a source file (good enough for bucketing)."""
    out = []
    pat = re.compile(r"^\s*(?:template\s*<[^>]*>\s*)?(?:UPKIE_HD|__global__|static|inline|__device__)[^;=]*?\b(\w+)\s*\(")
    lam = re.compile(r"^\s*auto\s+(\w+)\s*=\s*\[")
    for i, line in enumerate(open(path), 1):
        m = pat.match(line) or lam.match(line)
        if m and m.group(1) not in ("if", "for", "while", "return"):
            out.append((i, m.group(1)))
    return out


PHASE_MARKERS = [  # (regex on a source line of physics_substep_paired, phase that starts there)
    (r"float R\[9\];", "rotation, base inertia"),
    (r"legs_pass12\(P, S\.q", "ABA passes 1-2, both legs"),
    (r"ldl6\(IA0\);", "base LDL^T + solve"),
    (r"legs_pass3\(P, lc", "ABA pass 3"),
    (r"// gravity as a uniform frame acceleration", "velocity update"),
    (r"// -- collision detection", "collision detection"),
    (r"bool ten_rows = limits == 2;", "ten-row solver (joint-limit + contact rows: Delassus, setup, sweeps, apply)"),
    (r"// contact directions in base coordinates", "contact Jacobians, wheel velocities"),
    (r"// Delassus matrix W = J M\^-1 J\^T without", "Delassus matrix"),
    (r"// right-hand sides \(btMultiBodyConstraintSolver", "row setup"),
    (r"auto sweep = \[&\]", "PGS sweeps"),
    (r"for \(int it = 0; it < P\.pgs_iterations; it \+= 2\)", "PGS sweeps (two inlined copies of the six-row sweep, plain and with exit test) + loop control"),
    (r"// apply the total wheel impulses", "apply impulses"),
    (r"if \(slow\) limit_contact_solve", "joint-limit slow path"),
    (r"// -- position integration with the new velocities", "position integration"),
]


def ncu_rows(rep):
    """[(opcode text, executed warp instructions, {stall: samples})] per SASS instruction of the first kernel in rep."""
    import csv
    import io

    src = subprocess.run(["ncu", "-i", rep, "--page", "source", "--csv"], capture_output=True, text=True).stdout
    rows = list(csv.reader(io.StringIO(src)))
    hdr = rows[1]
    i_src, i_exe = hdr.index("Source"), hdr.index("Instructions Executed")
    stall_cols = [(i, h) for i, h in enumerate(hdr) if h.startswith("stall_") and "Not Issued" not in h]
    out = []
    for r in rows[2:]:
        if len(r) < len(hdr):
            if r and r[0] == "Kernel Name":
                break
            continue
        try:
            exe = int(r[i_exe])
        except ValueError:
            continue
        st = {}
        for i, h in stall_cols:
            try:
                v = int(r[i])
            except ValueError:
                v = 0
            if v:
                st[h] = v
        out.append((r[i_src].strip(), exe, st))
    return out


# H100: 256 KB of L1 + shared memory per SM, shared-memory carveout steps in KB, 1 KB reserved per block; the
# headline launch: one 256-thread block per SM (255 registers), one 36-float action tile row per thread
SM_L1_SMEM_KB = 256
CARVEOUTS_KB = [0, 8, 16, 32, 64, 100, 132, 164, 196, 228]
BLOCK = 256


def l1_budget(text):
    """the local-memory frame of a block against the L1 its smallest carveout leaves (launch_k_step: one tile buffer
    per warp when the block steps one tile, the carveout preference cudaSharedmemCarveoutMaxL1)"""
    frames = [int(v, 16) for v in re.findall(r"(?:IADD3|VIADD)\s+R1, R1, -0x([0-9a-f]+)", text)]
    frame = max(frames) if frames else 0
    ldl = len(re.findall(r"\bLDL\b", text))
    stl = len(re.findall(r"\bSTL\b", text))
    smem_kb = BLOCK * 36 * 4 / 1024 + 1
    carve = next(c for c in CARVEOUTS_KB if c >= smem_kb)
    l1_kb = SM_L1_SMEM_KB - carve
    need_kb = frame * BLOCK / 1024
    print(f"frame {frame} B x {BLOCK} threads = {need_kb:.0f} KB vs L1 left {l1_kb} KB (block {smem_kb:.0f} KB of "
          f"shared memory -> {carve} KB carveout): {'fits' if need_kb <= l1_kb else 'does NOT fit'}; "
          f"{ldl} LDL, {stl} STL")


def main():
    args = [a for a in sys.argv[1:]]
    rep = None
    if "--ncu" in args:
        k = args.index("--ncu")
        rep = args[k + 1]
        del args[k:k + 2]
    lib = LIB
    if "--lib" in args:
        k = args.index("--lib")
        lib = args[k + 1]
        del args[k:k + 2]
    want = args[0] if args else "k_stepILi0ELi1ELi2ELi1E"
    dyn = ncu_rows(rep) if rep else None
    # every step unit compiles step_unit.cu, so the cubins cuobjdump extracts from the library share one file name and
    # overwrite each other: extract them from the unit objects next to the library (build.py's build/) when they exist
    objdir = os.path.join(os.path.dirname(os.path.abspath(lib)), "build")
    objs = sorted(os.path.join(objdir, f) for f in os.listdir(objdir) if f.endswith(".o")) if os.path.isdir(objdir) else []
    with tempfile.TemporaryDirectory() as tmp:
        cubins = []
        for k, src in enumerate(objs or [lib]):
            d = os.path.join(tmp, str(k))
            os.makedirs(d)
            subprocess.run(["cuobjdump", "-xelf", "all", src], cwd=d, check=True, stdout=subprocess.DEVNULL)
            cubins += [os.path.join(d, c) for c in sorted(os.listdir(d))]
        text = None
        for cubin in cubins:
            dis = subprocess.run(["nvdisasm", "--print-line-info-inline", cubin],
                                 capture_output=True, text=True).stdout
            m = re.search(r"^\.text\.(\S*" + re.escape(want) + r"\S*):", dis, re.M)
            if m:
                start = m.end()
                nxt = re.search(r"^\.text\.\S+:", dis[start:], re.M)
                text = dis[start:start + nxt.start()] if nxt else dis[start:]
                print(f"kernel {m.group(1)[:90]}... in {cubin}")
                break
        if text is None:
            raise SystemExit(f"no kernel matching {want!r} in {lib}")
    starts = {}

    def func_of(fn, ln):
        if fn not in starts:
            p = os.path.join(CSRC, fn)
            starts[fn] = function_starts(p) if os.path.exists(p) else []
        name = "?"
        for s_line, s_name in starts[fn]:
            if s_line <= ln:
                name = s_name
            else:
                break
        return name

    # phases of physics_substep_paired by line
    pair_src = open(os.path.join(CSRC, "sim_pair.cuh")).read().splitlines()
    fn_start = next(i for i, l in enumerate(pair_src, 1) if "void physics_substep_paired(" in l)
    phase_lines = []
    for rx, name in PHASE_MARKERS:
        for i in range(fn_start, len(pair_src) + 1):
            if re.search(rx, pair_src[i - 1]):
                phase_lines.append((i, name))
                break
    phase_lines.sort()

    def phase_of(ln):
        name = "substep prologue"
        for s_line, s_name in phase_lines:
            if s_line <= ln:
                name = s_name
        return name

    counts, packed = collections.Counter(), collections.Counter()
    dyn_exe, dyn_stall = collections.Counter(), collections.defaultdict(collections.Counter)
    chain, total = [], 0
    pending = []
    for line in text.splitlines():
        m = re.match(r'\s*//## File "([^"]+)", line (\d+)(?: inlined at "([^"]+)", line (\d+))?', line)
        if m:
            pending.append((os.path.basename(m.group(1)), int(m.group(2))))
            if m.group(3):
                pending.append((os.path.basename(m.group(3)), int(m.group(4))))
            continue
        if re.match(r"\s+/\*[0-9a-f]{4,6}\*/\s+\S", line):
            if pending:
                chain, pending = pending, []
            frames = [(fn, ln, func_of(fn, ln)) for fn, ln in chain]  # innermost first
            bucket = None
            for fn, ln, name in reversed(frames):  # outermost first
                if fn == "sim_pair.cuh" and ln >= fn_start:  # physics_substep_paired is the last function of the file
                    bucket = "substep: " + phase_of(ln)
                    break
            if bucket is None:
                named = [name for fn, ln, name in reversed(frames) if fn.endswith((".cuh", ".cu", ".h"))
                         and name not in ("step_env", "k_step", "__launch_bounds__", "prefetch", "?")]
                bucket = "tick: " + (named[0] if named else "step_env (front-end, observation, stores)")
            counts[bucket] += 1
            if re.search(r"\b(FFMA2|FMUL2|FADD2)\b", line):
                packed[bucket] += 1
            if dyn is not None and total < len(dyn):
                op = re.search(r"\*/\s+(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", line)
                dop = re.match(r"(?:@!?U?P\d+\s+)?([A-Z0-9_.]+)", dyn[total][0])
                if op and dop and op.group(1).split(".")[0] != dop.group(1).split(".")[0]:
                    raise SystemExit(f"instruction {total}: library has {op.group(1)}, report has {dop.group(1)} - the "
                                     "ncu report is not from this build")
                dyn_exe[bucket] += dyn[total][1]
                for h, v in dyn[total][2].items():
                    dyn_stall[bucket][h] += v
            total += 1
    print(f"{total} static instructions ({sum(packed.values())} packed f32x2)")
    l1_budget(text)
    if dyn is None:
        print(f"{'instr':>6s} {'share':>6s} {'f32x2':>6s}  bucket")
        for bucket, c in sorted(counts.items(), key=lambda kv: (not kv[0].startswith("substep"), -kv[1])):
            print(f"{c:6d} {100.0 * c / total:5.1f}% {packed[bucket]:6d}  {bucket}")
        return
    if len(dyn) != total:
        print(f"WARNING: report has {len(dyn)} instructions, library kernel {total}")
    tot_exe = sum(dyn_exe.values())
    tot_smp = sum(sum(c.values()) for c in dyn_stall.values())
    print(f"dynamic: {tot_exe} warp instructions, {tot_smp} stall samples (time share ~ sample share)")
    print(f"{'static':>6s} {'dyn instr':>7s} {'samples':>7s}  top stall reasons                                   bucket")
    for bucket, c in sorted(counts.items(), key=lambda kv: -sum(dyn_stall[kv[0]].values())):
        smp = sum(dyn_stall[bucket].values())
        top = ", ".join(f"{h[6:]} {100.0 * v / max(1, smp):.0f}%" for h, v in dyn_stall[bucket].most_common(3))
        print(f"{c:6d} {100.0 * dyn_exe[bucket] / max(1, tot_exe):6.1f}% {100.0 * smp / max(1, tot_smp):6.1f}%  {top:50s}  {bucket}")


if __name__ == "__main__":
    main()
