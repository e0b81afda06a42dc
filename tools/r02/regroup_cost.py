#!/usr/bin/env python3
# SPDX-License-Identifier: Apache-2.0
"""Cost model of regrouping a block's robots by contact class before the contact solve (developer tool, no GPU).

Reads the per-robot-substep records of tools/r02/pgs_stats.cpp (uint8 [ticks][n][5]: 0 no solve, s six-row
sweeps, 100 + s ten-row sweeps, 255 idle lane of a reset tick) and predicts the warp-instructions of one tick for
  - today's per-warp choice (`joint_limits = 3`: ten-row solver if any lane is on a bound, six-row if any lane is
    in contact, none otherwise; a warp loops until its slowest lane is frozen, two sweeps per trip), and
  - the same choice after a stable counting sort of each block's robots by class (blocks of 128 and 256), plus the
    exchange through shared memory (ballots, counters, barriers, the solver's inputs and outputs).

    g++ -O2 -std=c++17 -DUPKIE_PGS_STATS -o pgs_stats tools/r02/pgs_stats.cpp   # model dump: see body_gate_stats.cpp
    ./pgs_stats 16384 200 > pgs.bin
    python tools/r02/regroup_cost.py pgs.bin 16384 [--skip 50]

The static sizes are those of `tools/static_breakdown.py` on the sm_90a build (override with --sizes k=v,...). The last
column bounds the other side: with one barrier per substep a block's solver phase lasts as long as its slowest warp.
"""
import argparse

import numpy as np

SIZES = {
    "common": 3250,  # substep outside the solver branches: torque law (831), ABA (1878 + 96), base LDL^T (145),
                     # rotation and base inertia (132), velocity update (70), collision (37), integration (61)
    "tick": 1800,    # per tick outside the substep loop: loads, front-end, observation, stores
    "ten_setup": 2023,  # ten-row branch without its sweep loop (2385 static - 362)
    "ten_trip": 362,    # one trip of the ten-row loop: two sweeps + exit vote
    "six_setup": 1115,  # six-row branch without its sweep loop: Jacobians 132, Delassus 572, rows 142, apply 260,
                        # loop control 9
    "six_trip": 177,    # one trip of the six-row loop
    "skip": 20,         # neither solver: zero the impulses
    "exchange": 320,    # per warp-substep of a regrouped block: class ballots + counting sort (~40), 117 input words
                        # stored and loaded, 18 output words stored and loaded, three barriers
}


def warp_cost(cls, sw, S):
    """Solver warp-instructions of warps given per-lane class [w][32] and sweeps [w][32]."""
    wc = cls.max(axis=1)
    trips = np.maximum(1, (sw.max(axis=1) + 1) // 2)
    return np.where(wc == 2, S["ten_setup"] + trips * S["ten_trip"],
                    np.where(wc == 1, S["six_setup"] + trips * S["six_trip"], S["skip"]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("records")
    ap.add_argument("n", type=int)
    ap.add_argument("--skip", type=int, default=50, help="ticks dropped as warm-up")
    ap.add_argument("--sizes", default="", help="k=v,... overrides of the static sizes")
    a = ap.parse_args()
    S = dict(SIZES)
    for kv in filter(None, a.sizes.split(",")):
        k, v = kv.split("=")
        S[k] = int(v)
    rec = np.fromfile(a.records, dtype=np.uint8).reshape(-1, a.n, 5)[a.skip:]
    ticks = rec.shape[0]
    idle = rec == 255
    cls = np.where(idle | (rec == 0), 0, np.where(rec >= 100, 2, 1)).astype(np.int8)
    sw = np.where(idle | (rec == 0), 0, np.where(rec >= 100, rec.astype(int) - 100, rec)).astype(np.int32)
    cls, sw = cls.transpose(0, 2, 1), sw.transpose(0, 2, 1)  # [tick][substep][robot]
    nwarps = a.n // 32
    shares = [np.mean(cls == c) for c in range(3)]
    print(f"{ticks} ticks x {a.n} robots: class 0 (no rows) {shares[0]:.1%}, class 1 (contact only) {shares[1]:.1%}, "
          f"class 2 (on a bound) {shares[2]:.1%}")

    fixed = nwarps * (S["tick"] + 5 * S["common"])  # per tick, the same in every arrangement

    def per_tick(block):
        c, s = cls, sw
        extra = 0
        if block:
            # stable counting sort by class inside each block of `block` robots (argsort is stable with kind="stable")
            cb = c.reshape(ticks, 5, -1, block)
            sb = s.reshape(ticks, 5, -1, block)
            order = np.argsort(cb, axis=-1, kind="stable")
            cb = np.take_along_axis(cb, order, -1)
            sb = np.take_along_axis(sb, order, -1)
            c, s = cb.reshape(ticks, 5, -1), sb.reshape(ticks, 5, -1)
            # blocks without a robot on a bound bypass the exchange
            has2 = (cls.reshape(ticks, 5, -1, block) == 2).any(-1)
            extra = S["exchange"] * (block // 32) * has2.sum() / ticks
        cw = c.reshape(ticks, 5, nwarps, 32)
        swp = s.reshape(ticks, 5, nwarps, 32)
        per_warp = warp_cost(cw.reshape(-1, 32), swp.reshape(-1, 32), S).reshape(ticks, 5, nwarps)
        solver = per_warp.sum() / ticks
        # the per-substep barriers make a block wait for its slowest warp: the solver phase of a block lasts as long
        # as its longest warp (at 2 warps per scheduler the others cannot fill the idle issue slots)
        wpb = (block or bound_block) // 32
        slowest = per_warp.reshape(ticks, 5, -1, wpb).max(-1).sum() * wpb / ticks
        wclass = cw.max(-1)
        trips = np.maximum(1, (swp.max(-1) + 1) // 2)
        return (fixed + solver + extra, solver, extra, np.mean(wclass == 2), np.mean(trips[wclass > 0] * 2),
                fixed + slowest + extra)

    rows = [("per-warp choice (today)", 0), ("block-sorted, 128", 128), ("block-sorted, 256", 256)]
    print(f"{'arrangement':<26s} {'warp-instr/tick':>15s} {'solver':>10s} {'exchange':>9s} {'ten-row warps':>13s} "
          f"{'sweeps/warp':>11s} {'vs today':>8s} {'slowest-warp bound vs today':>28s}")
    for bound_block in (128, 256):
        base = per_tick(0)
        for name, blk in rows:
            if blk and blk != bound_block:
                continue
            t, sol, ex, f10, swpw, slow = per_tick(blk)
            print(f"{name:<26s} {t:15.4g} {sol:10.4g} {ex:9.3g} {f10:13.1%} {swpw:11.2f} {t / base[0] - 1:+8.1%} "
                  f"{slow / base[5] - 1:+28.1%}" + ("" if blk else f"   ({bound_block}-thread blocks)"))


if __name__ == "__main__":
    main()
